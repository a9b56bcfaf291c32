"""ctypes binding of the C ABI (include/v2e_b200.h). Fails loudly: there is no CPU fallback."""
import ctypes
import os

from . import build as _build

_LIB = None


class V2eEmuCfg(ctypes.Structure):
    _fields_ = [
        ("width", ctypes.c_int32), ("height", ctypes.c_int32),
        ("per_pixel_thres", ctypes.c_int32), ("hdr", ctypes.c_int32),
        ("pos_thres_nominal", ctypes.c_double), ("neg_thres_nominal", ctypes.c_double),
        ("cutoff_hz", ctypes.c_double), ("leak_rate_hz", ctypes.c_double),
        ("leak_jitter_fraction", ctypes.c_double), ("refractory_period_s", ctypes.c_double),
        ("shot_noise_rate_hz", ctypes.c_double), ("shot_inten_factor", ctypes.c_double),
        ("rng_mode", ctypes.c_int32), ("iter_cap", ctypes.c_int32),
        ("seed", ctypes.c_uint64),
        ("csdvs", ctypes.c_int32), ("max_frames_per_step", ctypes.c_int32),
        ("cs_tau_p_s", ctypes.c_double), ("cs_tau_h_s", ctypes.c_double),
        ("scidvs", ctypes.c_int32), ("photoreceptor_noise", ctypes.c_int32),
        ("rng_pixel_offset", ctypes.c_uint32), ("full_frame_px", ctypes.c_uint32),
        ("own_row0", ctypes.c_int32), ("own_rows", ctypes.c_int32),
        ("cs_halo_rows", ctypes.c_int32), ("reserved1", ctypes.c_int32),
    ]


class V2eUNetWeights(ctypes.Structure):
    _fields_ = [("w", ctypes.c_void_p * 23), ("b", ctypes.c_void_p * 23)]


class V2eFrameInfo(ctypes.Structure):
    _fields_ = [
        ("max_n", ctypes.c_int32), ("filter_active", ctypes.c_int32),
        ("n_on", ctypes.c_uint32), ("n_off", ctypes.c_uint32),
        ("n_shot_on", ctypes.c_uint32), ("n_shot_off", ctypes.c_uint32),
        ("n_events", ctypes.c_uint32), ("cs_steps", ctypes.c_int32),
        ("ev_base", ctypes.c_uint64),
    ]


V2E_OK, V2E_E_INVALID, V2E_E_CUDA, V2E_E_CAPACITY, V2E_E_ITER_CAP, V2E_E_STATE, V2E_E_UNSUPPORTED, V2E_E_FALLBACK = \
    0, -1, -2, -3, -4, -5, -6, -7
ABI_VERSION = 201
U8, F32, F64 = 0, 1, 2

_vp, _i, _d, _u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_uint64

_SIGS = {
    "v2e_last_error": (ctypes.c_char_p, []),
    "v2e_version": (_i, []),
    "v2e_abi_info": (_i, [ctypes.POINTER(_i), ctypes.POINTER(_i), ctypes.POINTER(_i), ctypes.POINTER(_i)]),
    "v2e_emu_set_option": (_i, [_vp, _i, _i]),
    "v2e_emu_set_key_buffer": (_i, [_vp, _vp]),
    "v2e_emu_order_stats": (_i, [_vp, ctypes.POINTER(_u64), ctypes.POINTER(ctypes.c_longlong)]),
    "v2e_emu_fused_count": (_i, [_vp, _vp, _i, _i, _vp, _d, _vp]),
    "v2e_emu_max_vec_dev": (_vp, [_vp]),
    "v2e_emu_fused_emit": (_i, [_vp, _vp, _u64, _u64, _vp]),
    "v2e_emu_fused_stats": (_i, [_vp, ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_longlong)]),
    "v2e_emu_cs_paths": (_i, [_vp, ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_longlong)]),
    "v2e_emu_fused_frames": (_i, [_vp, ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_longlong)]),
    "v2e_emu_fused_last_reject": (_i, [_vp, ctypes.POINTER(_i), ctypes.POINTER(_i)]),
    "v2e_emu_time_fused": (_i, [_vp, _vp, _i, _i, _vp, _d, _vp, _u64, _i, ctypes.POINTER(ctypes.c_float),
                                ctypes.POINTER(ctypes.c_float), _vp]),
    "v2e_emu_create": (_i, [ctypes.POINTER(V2eEmuCfg), ctypes.POINTER(_vp)]),
    "v2e_emu_destroy": (_i, [_vp]),
    "v2e_emu_set_linlog_lut": (_i, [_vp, _vp, _vp]),
    "v2e_emu_set_fields": (_i, [_vp, _vp, _vp, _vp]),
    "v2e_emu_first_frame": (_i, [_vp, _vp, _i, _d, _d, _vp]),
    "v2e_emu_step": (_i, [_vp, _vp, _i, _i, _vp, _d, _vp, _vp, _vp, _u64, _u64, _i, _i, _vp]),
    "v2e_emu_collect": (_i, [_vp, ctypes.POINTER(V2eFrameInfo), _i, ctypes.POINTER(_i),
                             ctypes.POINTER(_u64), _vp]),
    "v2e_emu_phase_count": (_i, [_vp, _vp, _i, _d, _d, _vp, _vp, _i, _u64, _u64, _vp]),
    "v2e_emu_phase_update": (_i, [_vp, _vp, _i, _d, _d, _vp, _vp, _u64, _u64, _vp]),
    "v2e_emu_max_n_dev": (_vp, [_vp]),
    "v2e_emu_cs_begin": (_i, [_vp, _vp, _i, _d, _d, _u64, _u64, ctypes.POINTER(_i), _vp]),
    "v2e_emu_cs_pack": (_i, [_vp, _vp]),
    # the halo exchange buffers (send, rows above / below) hold the state dtype: float64, or float32 at cutoff_hz = 0
    "v2e_emu_cs_unpack_from": (_i, [_vp, _vp, _vp, _vp]),
    "v2e_emu_cs_send_dev": (_vp, [_vp]),
    "v2e_emu_cs_chunk": (_i, [_vp, _i, _i, _vp]),
    "v2e_emu_cs_max_dev": (_vp, [_vp]),
    "v2e_emu_cs_advance": (_i, [_vp, _i, _i, _vp]),
    "v2e_emu_cs_update": (_i, [_vp, _vp, _i, _vp, _vp, _vp]),
    "v2e_emu_phase_filter": (_i, [_vp, _d, _d, _u64, _i, _vp]),
    "v2e_emu_read_counts": (_i, [_vp, ctypes.POINTER(ctypes.c_int32), _vp, _i, _vp]),
    "v2e_emu_phase_shot": (_i, [_vp, _vp, _i, _d, _d, _vp, _u64, _vp]),
    "v2e_emu_phase_emit": (_i, [_vp, _d, _d, _vp, _u64, _vp]),
    "v2e_conv2d_lrelu_sm100": (_i, [_vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _i,
                                    ctypes.c_float, _vp]),
    "v2e_conv2d_lrelu_sm100_tile": (_i, [_vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _i,
                                         ctypes.c_float, _i, _i, _vp]),
    "v2e_conv_pick_tile": (_i, [_i, _i, _i, _i, _i, _i, _i, _i, _i]),
    "v2e_conv2d_lrelu_sm100_strip": (_i, [_vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _i,
                                          ctypes.c_float, _vp]),
    "v2e_conv_strip_pick_kc": (_i, [_i, _i, _i, _i, _i, _i]),
    "v2e_conv2d_up2_lrelu_sm100": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _i, ctypes.c_float, _vp]),
    "v2e_conv_up2_fold_weights": (_i, [_vp, _i, _i, _i, _i, _vp]),
    "v2e_conv_up2_supported_c": (_i, [_i, _i, _i]),
    "v2e_slomo_create": (_i, [_i, _i, _i, _vp, _vp, ctypes.POINTER(_vp)]),
    "v2e_slomo_destroy": (_i, [_vp]),
    "v2e_slomo_set_pairs": (_i, [_vp, _vp, _i, _vp]),
    "v2e_slomo_max_flow": (_i, [_vp, ctypes.POINTER(ctypes.c_float), _vp]),
    "v2e_slomo_interp": (_i, [_vp, _d, _vp, _vp, _vp]),
    "v2e_slomo_set_option": (_i, [_vp, _i, _i]),
    "v2e_slomo_check_finite": (_i, [_vp, ctypes.POINTER(_i), _vp]),
    "v2e_slomo_profile": (_i, [_vp, _i]),
    "v2e_slomo_profile_read": (_i, [_vp, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(_i),
                                    ctypes.POINTER(ctypes.c_double), _vp]),
    "v2e_slomo_profile_read_layers": (_i, [_vp, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(_i),
                                           ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_float),
                                           ctypes.POINTER(_i), ctypes.POINTER(ctypes.c_double), _vp]),
    "v2e_slomo_flow_ptr": (_vp, [_vp]),
    "v2e_slomo_intrp_ptr": (_vp, [_vp]),
    "v2e_slomo_buffer_ptr": (_vp, [_vp, _i, _i]),
    "v2e_slomo_layer_kernel": (_i, [_vp, _i, _i]),
    "v2e_resize_create": (_i, [_i, _i, _i, _i, _i, _i, ctypes.POINTER(_vp)]),
    "v2e_resize_destroy": (_i, [_vp]),
    "v2e_resize_run": (_i, [_vp, _vp, _vp, _i, _vp]),
    "v2e_resize_run_strided": (_i, [_vp, _vp, _vp, _i, ctypes.c_long, _vp]),
    "v2e_emu_set_scidvs_tau": (_i, [_vp, _vp]),
    "v2e_emu_set_pr_noise": (_i, [_vp, _vp, ctypes.POINTER(_d), _i]),
    "v2e_prep_create": (_i, [_i, _i, _i, _i, _i, _i, _i, _i, _i, ctypes.POINTER(_vp)]),
    "v2e_prep_destroy": (_i, [_vp]),
    "v2e_prep_run": (_i, [_vp, _vp, _i, _vp, _vp]),
    "v2e_render_area_scan": (_i, [_vp, ctypes.c_int64, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp]),
    "v2e_render_frames": (_i, [_vp, _vp, _vp, _i, ctypes.c_int64, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "v2e_events_to_h5_rows": (_i, [_vp, _u64, _vp, _vp]),
    "v2e_events_to_aedat2": (_i, [_vp, _u64, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "v2e_events_to_text_scratch": (_u64, [_u64]),
    "v2e_events_to_text_layout": (_i, [_vp, _u64, _vp, _vp, _vp]),
    "v2e_events_to_text": (_i, [_vp, _u64, _vp, _vp, _vp, _vp]),
    "v2e_signnoise_labels": (_i, [_vp, _vp, _i, _u64, _vp, _vp]),
    "v2e_emu_profile": (_i, [_vp, _i]),
    "v2e_emu_profile_read4": (_i, [_vp, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(_i), _vp]),
    "v2e_emu_state_is_f64": (_i, [_vp]),
    "v2e_emu_state_ptr": (_vp, [_vp, _i]),
    "v2e_emu_draw_noise": (_i, [_vp, ctypes.c_uint32, _vp, _vp, _vp, _vp]),
}


def library_path():
    return _build.LIB


def load(build_if_missing=True):
    """Loads libv2e_b200.so (building it with nvcc if the in-tree copy is missing or stale)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = _build.LIB
    if build_if_missing and os.environ.get("V2E_B200_NO_BUILD") != "1":
        try:
            _build.build()
        except Exception as e:  # a present library may still be current (checked below); a missing one is fatal
            if not os.path.exists(path):
                raise RuntimeError("v2e_b200: the CUDA library is not built and nvcc failed: %s" % e)
            import warnings
            warnings.warn("v2e_b200: rebuilding %s failed (%s); using the existing library if its ABI matches"
                          % (path, e))
    if not os.path.exists(path):
        raise RuntimeError("v2e_b200: %s is missing -- run `python -m v2e_b200.build`; "
                           "there is no CPU fallback" % path)
    lib = ctypes.CDLL(path)
    missing = [name for name in _SIGS if not hasattr(lib, name)]
    if missing:
        raise RuntimeError("v2e_b200: %s is stale (missing %s) -- rebuild with `python -m v2e_b200.build --force`"
                           % (path, ", ".join(missing[:6])))
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    # the ctypes structs above must be the layouts the library was compiled with
    ver, a, b, c = _i(0), _i(0), _i(0), _i(0)
    lib.v2e_abi_info(ctypes.byref(ver), ctypes.byref(a), ctypes.byref(b), ctypes.byref(c))
    want = (ABI_VERSION, ctypes.sizeof(V2eEmuCfg), ctypes.sizeof(V2eFrameInfo), ctypes.sizeof(V2eUNetWeights))
    if (ver.value, a.value, b.value, c.value) != want:
        raise RuntimeError("v2e_b200: %s has ABI %s, this binding expects %s -- rebuild with "
                           "`python -m v2e_b200.build --force`" % (path, (ver.value, a.value, b.value, c.value), want))
    _LIB = lib
    return lib


class V2eError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("v2e_b200 error %d: %s" % (code, msg))
        self.code = code


def check(rc):
    if rc != 0:
        raise V2eError(rc, load().v2e_last_error().decode(errors="replace"))
    return rc
