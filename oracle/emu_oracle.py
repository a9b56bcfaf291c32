"""TEST INFRASTRUCTURE ONLY -- Python driver of the scalar C oracle (emu_oracle.c).

Not part of the product: v2e_b200/ never imports this. Only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs do.

Mirrors the call contract of the reference's EventEmulator.generate_events
(/root/reference/v2ecore/emulator.py:619-1022) closely enough that parity tests read
like "same inputs, same seed -> same rows". All random draws use torch's global CPU
generator with the same calls in the same order as the reference (SURVEY.md 7,
"RNG parity"): _init: normal(pos), normal(neg), [randn noise_rate]; every later
frame: [randn leak], randperm(n_i) per iteration that has events, [rand shot].
"""
import ctypes
import math
import os
import subprocess

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class _Cfg(ctypes.Structure):
    _fields_ = [
        ("width", ctypes.c_int32), ("height", ctypes.c_int32),
        ("state_f64", ctypes.c_int32), ("per_pixel_thres", ctypes.c_int32),
        ("hdr", ctypes.c_int32), ("frame_dtype", ctypes.c_int32),
        ("pos_thres_nominal", ctypes.c_double), ("neg_thres_nominal", ctypes.c_double),
        ("cutoff_hz", ctypes.c_double),
        ("leak_rate_hz", ctypes.c_double), ("leak_jitter_fraction", ctypes.c_double),
        ("refractory_period_s", ctypes.c_double),
        ("shot_noise_rate_hz", ctypes.c_double),
        ("shot_inten_factor", ctypes.c_double),
        ("csdvs", ctypes.c_int32), ("_pad", ctypes.c_int32),
        ("cs_tau_p_s", ctypes.c_double), ("cs_tau_h_s", ctypes.c_double),
        ("scidvs", ctypes.c_int32), ("pr_noise", ctypes.c_int32),
        ("scidvs_first", ctypes.c_int32), ("_pad2", ctypes.c_int32),
        ("pr_vrms", ctypes.c_double),
    ]


class _State(ctypes.Structure):
    _fields_ = [
        ("lp", ctypes.c_void_p), ("base", ctypes.c_void_p),
        ("pos_thres", ctypes.c_void_p), ("neg_thres", ctypes.c_void_p),
        ("noise_rate", ctypes.c_void_p), ("tmem", ctypes.c_void_p),
        ("surround", ctypes.c_void_p), ("linlog_lut", ctypes.c_void_p),
        ("hp", ctypes.c_void_p), ("prev_photo", ctypes.c_void_p), ("tau_arr", ctypes.c_void_p),
        ("noise_arr", ctypes.c_void_p), ("pr_randn", ctypes.c_void_p),
    ]


def build_oracle(force=False):
    so = os.path.join(_HERE, "libemu_oracle.so")
    src = os.path.join(_HERE, "emu_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-B", "libemu_oracle.so"],
                              stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build_oracle())
        L.oracle_emu_first_frame.restype = ctypes.c_int
        L.oracle_emu_first_frame.argtypes = [ctypes.POINTER(_Cfg), ctypes.POINTER(_State),
                                             ctypes.c_void_p, ctypes.c_double, ctypes.c_double]
        L.oracle_emu_frame.restype = ctypes.c_long
        L.oracle_emu_frame.argtypes = [ctypes.POINTER(_Cfg), ctypes.POINTER(_State), ctypes.c_void_p,
                                       ctypes.c_double, ctypes.c_double, ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_long, ctypes.c_void_p, ctypes.c_long,
                                       ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.oracle_emu_shot.restype = ctypes.c_long
        L.oracle_emu_shot.argtypes = [ctypes.POINTER(_Cfg), ctypes.POINTER(_State), ctypes.c_void_p,
                                      ctypes.c_double, ctypes.c_double, ctypes.c_int32, ctypes.c_void_p,
                                      ctypes.c_void_p, ctypes.c_long, ctypes.c_void_p]
        L.oracle_linspace_f32.restype = ctypes.c_float
        L.oracle_linspace_f32.argtypes = [ctypes.c_double, ctypes.c_double, ctypes.c_int64, ctypes.c_int64]
        L.oracle_lap_kernel_order.restype = ctypes.c_int
        L.oracle_lap_kernel_order.argtypes = [ctypes.c_long, ctypes.c_long, ctypes.c_long]
        L.oracle_laplacian_f32.restype = None
        L.oracle_laplacian_f32.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.c_long, ctypes.c_void_p]
        L.oracle_set_cs_perturbation.restype = None
        L.oracle_set_cs_perturbation.argtypes = [ctypes.c_int, ctypes.c_int]
        _LIB = L
    return _LIB


def linlog_lut():
    """256-entry float32 table of lin_log(0..255), evaluated with the reference's own
    torch expression (emulator_utils.py:18-45) so that it is exact by construction."""
    x = torch.arange(256, dtype=torch.float64)
    f = (1. / 20) * math.log(20)
    y = torch.where(x <= 20, x * f, torch.log(x))
    y = torch.round(y * 1e8) / 1e8
    return y.float().numpy().copy()


class TorchGlobalRNG:
    """Default draw source: torch's global CPU generator, same calls as the reference."""

    def normal(self, mean, std, shape):
        return torch.normal(mean, std, size=shape, dtype=torch.float32)

    def randn(self, shape):
        return torch.randn(shape, dtype=torch.float32)

    def rand(self, shape):
        return torch.rand(shape, dtype=torch.float32)

    def randperm(self, n):
        return torch.randperm(n)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


_vn_cache = {"rate": None, "vn": None}


def photoreceptor_noise_vrms(shot_noise_rate_hz, f3db, sample_rate_hz, pos_thr, neg_thr, sigma_thr):
    """Restatement of emulator_utils.py:177-295 (host-side numpy calibration of the Gaussian noise amplitude
    that yields the requested shot-noise rate after the RC low-pass). Like the reference it draws from an
    UNSEEDED numpy generator and caches the value per sample rate (+-10 %), so two runs differ in the last
    digits: parity tests take the reference's values from the fixture instead."""
    if _vn_cache["rate"] is not None and abs(sample_rate_hz / _vn_cache["rate"] - 1) < 0.1:
        return _vn_cache["vn"]
    x = math.log10((shot_noise_rate_hz / f3db) / 2)
    y = -0.0026 * x ** 3 - 0.036 * x ** 2 - 0.1949 * x + 0.321
    N = 300
    pos = pos_thr + sigma_thr * np.random.default_rng().standard_normal(N)
    neg = neg_thr + sigma_thr * np.random.default_rng().standard_normal(N)
    vn = float(np.mean(np.minimum(pos, neg) / (10 ** y)))
    tau = 1 / (f3db * 2 * math.pi)
    dt = 1 / sample_rate_hz
    t = np.arange(0, 1000 * tau, dt)
    rin = vn * np.random.default_rng().standard_normal(t.shape)
    eps = dt / tau
    rout = np.zeros_like(rin)
    for i in range(1, len(rin)):
        rout[i] = rout[i - 1] * (1 - eps) + rin[i] * eps
    scaled = float(np.std(rin) / np.std(rout) * vn)
    _vn_cache["rate"], _vn_cache["vn"] = sample_rate_hz, scaled
    return scaled


class OracleEmulator:
    """CPU oracle with the reference's constructor defaults (emulator.py:86-117)."""

    def __init__(self, pos_thres=0.2, neg_thres=0.2, sigma_thres=0.03, cutoff_hz=0.0,
                 leak_rate_hz=0.1, refractory_period_s=0.0, shot_noise_rate_hz=0.0,
                 leak_jitter_fraction=0.1, noise_rate_cov_decades=0.1, seed=0,
                 cs_lambda_pixels=None, cs_tau_p_ms=None, hdr=False, shuffle=True, rng=None,
                 scidvs=False, photoreceptor_noise=False, pr_vrms_tape=None):
        self.pos_thres_nominal, self.neg_thres_nominal = pos_thres, neg_thres
        self.sigma_thres = sigma_thres
        self.cutoff_hz = cutoff_hz
        self.leak_rate_hz = leak_rate_hz
        self.refractory_period_s = refractory_period_s
        self.shot_noise_rate_hz = shot_noise_rate_hz
        self.leak_jitter_fraction = leak_jitter_fraction
        self.noise_rate_cov_decades = noise_rate_cov_decades
        self.hdr = hdr
        self.shuffle = shuffle
        self.rng = rng if rng is not None else TorchGlobalRNG()
        self.scidvs, self.photoreceptor_noise = scidvs, photoreceptor_noise
        self.pr_vrms_tape = list(pr_vrms_tape) if pr_vrms_tape is not None else None
        self.hp = self.prev_photo = self.tau_arr = self.noise_arr = None
        self._scidvs_started = False
        self._pr_randn = None
        self._pr_vrms = 0.0
        self.cs_lambda_pixels, self.cs_tau_p_ms = cs_lambda_pixels, cs_tau_p_ms
        self.csdvs = cs_lambda_pixels is not None
        if self.csdvs:
            self.cs_tau_h_ms = 0 if (cs_tau_p_ms is None or cs_tau_p_ms == 0) \
                else cs_tau_p_ms / (cs_lambda_pixels ** 2)
        if seed != 0:
            torch.manual_seed(seed)
            np.random.seed(seed)
        self.t_previous = 0
        self.frame_counter = 0
        self.num_events_total = self.num_events_on = self.num_events_off = 0
        self.base = None
        self.cs_steps_taken = []
        self.last_max_n = 0
        self._lut = linlog_lut()

    # -- helpers ---------------------------------------------------------
    def _frame_arg(self, new_frame):
        if isinstance(new_frame, torch.Tensor):
            new_frame = new_frame.cpu().numpy()
        a = np.ascontiguousarray(new_frame)
        if a.dtype == np.uint8:
            return a, 0
        if a.dtype == np.float32:
            return a, 1
        return np.ascontiguousarray(a, dtype=np.float64), 2

    def _make_cfg(self, H, W, dtype):
        c = _Cfg()
        c.width, c.height = W, H
        c.state_f64 = 1 if self.state_f64 else 0
        c.per_pixel_thres = 1 if self.sigma_thres > 0 else 0
        c.hdr = 1 if self.hdr else 0
        c.frame_dtype = dtype
        c.pos_thres_nominal, c.neg_thres_nominal = self.pos_thres_nominal, self.neg_thres_nominal
        c.cutoff_hz = self.cutoff_hz
        c.leak_rate_hz, c.leak_jitter_fraction = self.leak_rate_hz, self.leak_jitter_fraction
        c.refractory_period_s = self.refractory_period_s
        c.shot_noise_rate_hz = self.shot_noise_rate_hz
        c.shot_inten_factor = 0.25
        c.csdvs = 1 if self.csdvs else 0
        if self.csdvs:
            abs_min = 1e-9
            c.cs_tau_p_s = abs_min if (self.cs_tau_p_ms is None or self.cs_tau_p_ms == 0) \
                else self.cs_tau_p_ms * 1e-3
            c.cs_tau_h_s = abs_min / (self.cs_lambda_pixels ** 2) \
                if (self.cs_tau_h_ms is None or self.cs_tau_h_ms == 0) else self.cs_tau_h_ms * 1e-3
        c.scidvs = 1 if self.scidvs else 0
        c.pr_noise = 1 if self.photoreceptor_noise else 0
        c.scidvs_first = 1 if (self.scidvs and not self._scidvs_started) else 0
        c.pr_vrms = float(self._pr_vrms)
        return c

    def _make_state(self):
        s = _State()
        s.lp, s.base = _ptr(self.lp), _ptr(self.base)
        s.pos_thres, s.neg_thres = _ptr(self.pos_thres), _ptr(self.neg_thres)
        s.noise_rate, s.tmem = _ptr(self.noise_rate), _ptr(self.tmem)
        s.surround = _ptr(self.surround)
        s.linlog_lut = _ptr(self._lut)
        s.hp, s.prev_photo, s.tau_arr = _ptr(self.hp), _ptr(self.prev_photo), _ptr(self.tau_arr)
        s.noise_arr, s.pr_randn = _ptr(self.noise_arr), _ptr(self._pr_randn)
        return s

    # -- API ---------------------------------------------------------------
    def generate_events(self, new_frame, t_frame):
        t_frame = float(t_frame)
        self.frame_counter += 1
        if t_frame < self.t_previous:
            raise ValueError("this frame time={} must be later than previous frame time={}".format(
                t_frame, self.t_previous))
        frame, dtype = self._frame_arg(new_frame)
        H, W = frame.shape
        L = lib()
        if self.base is None:
            self.state_f64 = self.cutoff_hz > 0 or self.hdr
            sdt = np.float64 if self.state_f64 else np.float32
            self.lp = np.zeros((H, W), sdt)
            self.base = np.zeros((H, W), sdt)
            self.surround = np.zeros((H, W), np.float64) if self.csdvs else None
            self.pos_thres = self.neg_thres = self.noise_rate = self.tmem = None
            cfg = self._make_cfg(H, W, dtype)
            st = self._make_state()
            L.oracle_emu_first_frame(cfg, st, _ptr(frame), t_frame, float(self.t_previous))
            # _init (emulator.py:439-511): draw order normal(pos), normal(neg), randn(noise_rate)
            if self.sigma_thres > 0:
                p = self.rng.normal(self.pos_thres_nominal, self.sigma_thres, (H, W))
                self.pos_thres = torch.clamp(p, min=0.01).numpy().copy()
                q = self.rng.normal(self.neg_thres_nominal, self.sigma_thres, (H, W))
                self.neg_thres = torch.clamp(q, min=0.01).numpy().copy()
            if self.scidvs:     # emulator.py:480-483: SCIDVS_TAU_S * exp(normal(0, SCIDVS_TAU_COV))
                self.tau_arr = (0.01 * torch.exp(self.rng.normal(0, 0.5, (H, W)))).numpy().copy()
                self.hp = np.zeros((H, W), sdt)
                self.prev_photo = np.zeros((H, W), sdt)
            if self.photoreceptor_noise:
                self.noise_arr = np.zeros((H, W), np.float32)     # zeros_like(float32 log frame), emulator.py:684
            if self.leak_rate_hz > 0:
                r = self.rng.randn((H, W))
                self.noise_rate = torch.exp(math.log(10) * self.noise_rate_cov_decades * r).numpy().copy()
            if self.refractory_period_s > 0:
                self.tmem = (torch.zeros((H, W), dtype=torch.float32) - self.refractory_period_s).numpy().copy()
            # NOTE: t_previous is NOT advanced on the first frame (emulator.py:717 returns early)
            return None

        if self.photoreceptor_noise:    # emulator.py:694-698: vrms, then the randn draw, before the leak draw
            dt = t_frame - self.t_previous
            if self.pr_vrms_tape is not None:
                self._pr_vrms = float(self.pr_vrms_tape.pop(0))
            else:
                self._pr_vrms = photoreceptor_noise_vrms(self.shot_noise_rate_hz, self.cutoff_hz, 1 / dt,
                                                         self.pos_thres_nominal, self.neg_thres_nominal,
                                                         self.sigma_thres)
            self._pr_randn = np.ascontiguousarray(self.rng.randn((H, W)).numpy())
        cfg = self._make_cfg(H, W, dtype)
        st = self._make_state()
        n = H * W
        leak = None
        if self.leak_rate_hz > 0:
            leak = np.ascontiguousarray(self.rng.randn((H, W)).numpy())
        cap = 4 * n + 1024
        iter_cap = 4096
        snap_arrs = (self.lp, self.base, self.tmem, self.surround, self.hp, self.prev_photo, self.noise_arr)
        snap = [x.copy() if x is not None else None for x in snap_arrs]
        while True:
            ev = np.empty((cap, 4), np.float32)
            iters = np.zeros(2 * iter_cap, np.int32)
            max_n = ctypes.c_int32(0)
            cs_steps = ctypes.c_int32(0)
            rows = L.oracle_emu_frame(cfg, st, _ptr(frame), t_frame, float(self.t_previous), _ptr(leak),
                                      _ptr(ev), cap, _ptr(iters), iter_cap, ctypes.byref(max_n),
                                      None, None, ctypes.byref(cs_steps))
            if rows >= 0:
                break
            # output buffer too small: restore the state and retry with more room
            for dst, src in zip(snap_arrs, snap):
                if dst is not None:
                    dst[...] = src
            cap *= 4
            iter_cap = max(iter_cap, max_n.value + 1)
        if self.csdvs:
            self.cs_steps_taken.append(cs_steps.value)
        self._scidvs_started = True
        self.last_max_n = max_n.value
        # signal rows (ON, OFF) of every iteration of this frame, empty ones included
        self.last_iter_counts = iters[:2 * max_n.value].reshape(-1, 2).copy()
        ev = ev[:rows]
        # replay the per-iteration shuffles (emulator.py:866-870)
        out = []
        off = 0
        for it in range(max_n.value):
            c_on, c_off = int(iters[2 * it]), int(iters[2 * it + 1])
            k = c_on + c_off
            if k > 0:
                blk = ev[off:off + k]
                idx = self.rng.randperm(k).numpy()
                out.append(blk[idx] if self.shuffle else blk)
                self.num_events_on += c_on
                self.num_events_off += c_off
                self.num_events_total += k
            off += k
        if self.shot_noise_rate_hz > 0 and not self.photoreceptor_noise:     # emulator.py:893
            rnd = np.ascontiguousarray(self.rng.rand((H, W)).numpy())
            sev = np.empty((2 * n, 4), np.float32)
            cnt = np.zeros(2, np.int32)
            srows = L.oracle_emu_shot(cfg, st, _ptr(frame), t_frame, float(self.t_previous), max_n.value,
                                      _ptr(rnd), _ptr(sev), 2 * n, _ptr(cnt))
            if srows > 0:
                out.append(sev[:srows])
                self.num_events_on += int(cnt[0])
                self.num_events_off += int(cnt[1])
                self.num_events_total += int(srows)
        self.t_previous = t_frame
        if out:
            return np.concatenate(out, axis=0)
        return None
