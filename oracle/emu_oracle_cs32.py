"""TEST INFRASTRUCTURE ONLY -- Python driver of emu_oracle_cs32.c: the CPU oracle with the centre-surround model on a
float32 photoreceptor state (cutoff_hz = 0). Not part of the product: v2e_b200/ never imports this.

OracleEmulatorCS32 is emu_oracle.OracleEmulator -- same constructor, draws and call contract -- running on the library
built from emu_oracle_cs32.c, which exports emu_oracle.c's entry points and adds the float32 surround. The surround
array has the state dtype, as the reference's clone of lp_log_frame does (emulator.py:1063).
"""
import ctypes
import os
import subprocess

import numpy as np

import emu_oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build_oracle_cs32(force=False):
    so = os.path.join(_HERE, "libemu_oracle_cs32.so")
    srcs = [os.path.join(_HERE, f) for f in ("emu_oracle_cs32.c", "emu_oracle.c")]
    if force or not os.path.exists(so) or any(os.path.getmtime(so) < os.path.getmtime(s) for s in srcs):
        # the flags of oracle/Makefile: no multiply-add may be contracted
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall",
                               "-o", so, srcs[0], "-lm"], cwd=_HERE)
    return so


def lib():
    """The float32 centre-surround oracle library, with emu_oracle.lib()'s argument types."""
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build_oracle_cs32())
        base = emu_oracle.lib()
        for name in ("oracle_emu_first_frame", "oracle_emu_frame", "oracle_emu_shot", "oracle_set_cs_perturbation"):
            getattr(L, name).restype = getattr(base, name).restype
            getattr(L, name).argtypes = getattr(base, name).argtypes
        L.oracle_set_cs_f64_rule.restype = None
        L.oracle_set_cs_f64_rule.argtypes = [ctypes.c_int]
        _LIB = L
    return _LIB


class OracleEmulatorCS32(emu_oracle.OracleEmulator):
    """emu_oracle.OracleEmulator on emu_oracle_cs32.c; a float32 state keeps a float32 surround."""

    def set_dvs_params(self, model):
        """The 'clean' preset (emulator.py:513-523) before the first frame. Like the reference it leaves the nominal
        thresholds that _init draws around as they are."""
        if model != "clean":
            raise ValueError("only the 'clean' preset is restated")
        self.sigma_thres = 0.02
        self.cutoff_hz = 0
        self.leak_rate_hz = self.leak_jitter_fraction = self.noise_rate_cov_decades = 0
        self.shot_noise_rate_hz = 0
        self.refractory_period_s = 0

    def _make_state(self):
        if self.surround is not None and self.surround.dtype != self.lp.dtype:
            self.surround = np.zeros_like(self.lp)        # first frame: the surround is a clone of lp
        return super()._make_state()

    def generate_events(self, new_frame, t_frame):
        # emu_oracle.OracleEmulator.generate_events calls emu_oracle.lib(): hand it this library for the call
        saved = emu_oracle._LIB
        emu_oracle._LIB = lib()
        try:
            return super().generate_events(new_frame, t_frame)
        finally:
            emu_oracle._LIB = saved
