"""The reference's model-state display (v2ecore/emulator.py:41-50, 580-617) restated in numpy: the display ranges,
the normalisation, the uint8 cast and the text overlay. Used by tests/test_model_states.py to check the fixtures made
by oracle/make_golden_model_states.py and the device's planes."""
import numpy as np

L255 = np.log(255)                      # a NumPy float64 scalar: under NEP 50 the float32 states normalise in float64
GR, LG, SLG = (0, 255), (0, L255), (-L255 / 8, L255 / 8)
RANGES = {'new_frame': GR, 'log_new_frame': LG, 'lp_log_frame': LG, 'scidvs_highpass': SLG,
          'photoreceptor_noise_arr': SLG, 'cs_surround_frame': LG, 'c_minus_s_frame': SLG,
          'base_log_frame': SLG, 'diff_frame': SLG}


def u8(v):
    """ndarray.astype(np.uint8) of float64 values on x86-64: truncation toward zero to int32, low 8 bits kept; NaN,
    +-inf and values outside int32 range give 0."""
    v = np.asarray(v, np.float64)
    out = np.zeros(v.shape, np.uint8)
    ok = (v > -2147483649.0) & (v < 2147483648.0)
    out[ok] = (np.trunc(v[ok]).astype(np.int64) & 0xFF).astype(np.uint8)
    return out


def normalise(x, name):
    """emulator.py:594-596: the float image before the overlay."""
    lo, hi = RANGES[name]
    return (np.asarray(x) - lo) / (hi - lo)


def plane(x, name):
    """The bytes of state `x` before the overlay: (img * 255).astype(np.uint8) of the normalised image."""
    return u8(normalise(x, name) * 255)


def overlay_text(frame_counter, t_previous):
    return f'fr:{frame_counter} t:{t_previous:.4f}s'


def overlay(plane_u8, frame_counter, t_previous, output_height):
    """emulator.py:609-612 on the bytes: putText draws 0.0 and 255.0 into the float image, which the x255 cast turns
    into 0 and 1, so colours 0 and 1 drawn into the bytes give the written frame (one channel of GRAY2BGR)."""
    import cv2
    img = np.ascontiguousarray(plane_u8).copy()
    text = overlay_text(frame_counter, t_previous)
    cv2.putText(img, text, org=(0, output_height), fontScale=1.3, color=(0, 0, 0),
                fontFace=cv2.FONT_HERSHEY_PLAIN, thickness=1)
    cv2.putText(img, text, org=(1, output_height - 1), fontScale=1.3, color=(1, 1, 1),
                fontFace=cv2.FONT_HERSHEY_PLAIN, thickness=1)
    return img
