"""GPU parity tests of the SuperSloMo path: wgmma conv kernels, UNet, warps/blend, Pillow-exact
resizes and the SuperSloMo drop-in, against the float32 torch reference (oracle/slomo_ref.py) and
the fixtures produced by the unmodified reference classes.

Floating-point path. The CUDA kernels use fp16 operands with fp32 accumulation (same 10-bit
mantissa as the TF32 tensor-core math the reference's cuDNN convolutions use by default on
Ampere+); tolerances are stated per test."""
import ctypes
import os

import numpy as np
import pytest
import torch

import slomo_ref
from helpers import GOLDEN_DIR, conv_bound, conv_ref64, err_ratio

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _lib():
    from v2e_b200 import _lib as L
    return L, L.load()


def pad16(c):
    return (c + 15) // 16 * 16


def cout_pad(c):
    p = pad16(c)
    return 16 if p <= 16 else 32 if p <= 32 else 64 if p <= 64 else (p + 127) // 128 * 128


def to_nhwc16(x):
    N, C, H, W = x.shape
    out = torch.zeros((N, H, W, pad16(C)), dtype=torch.float16, device=x.device)
    out[..., :C] = x.permute(0, 2, 3, 1).half()
    return out.contiguous()


def pack_w(w, C1, C2):
    Cout, Cin, KH, KW = w.shape
    C1p, C2p = pad16(C1), (pad16(C2) if C2 else 0)
    Cp = cout_pad(Cout)
    out = torch.zeros((Cp, KH * KW, C1p + C2p), dtype=torch.float16, device=w.device)
    wt = w.permute(0, 2, 3, 1).reshape(Cout, KH * KW, Cin).half()
    out[:Cout, :, :C1] = wt[:, :, :C1]
    if C2:
        out[:Cout, :, C1p:C1p + C2] = wt[:, :, C1:]
    return out.reshape(Cp, -1).contiguous(), Cp


CONV_CASES = [
    # N, H, W, C1, C2, Cout, K, out_mode
    (1, 8, 16, 64, 0, 64, 3, 0), (1, 8, 16, 64, 0, 64, 1, 0), (2, 17, 23, 64, 0, 32, 3, 0),
    (1, 32, 32, 32, 0, 32, 7, 0), (1, 32, 48, 32, 0, 64, 5, 0), (1, 16, 32, 2, 0, 32, 7, 0),
    (1, 16, 32, 12, 0, 32, 7, 0), (1, 8, 10, 512, 0, 512, 3, 0), (1, 16, 20, 512, 512, 512, 3, 0),
    (1, 64, 80, 32, 32, 32, 3, 0), (1, 32, 40, 64, 64, 64, 3, 0), (1, 32, 32, 32, 0, 5, 3, 1),
    (1, 32, 32, 32, 0, 4, 3, 1), (2, 64, 96, 256, 0, 128, 3, 0), (1, 5, 7, 128, 0, 256, 3, 0),
    # BN = 128 with two / four output-channel blocks on the co_fast grid (blocks of one pixel tile side by side),
    # grids of several waves; concatenated 256 + 256 input
    (4, 88, 160, 128, 0, 256, 3, 0), (8, 44, 80, 256, 256, 512, 3, 0), (8, 41, 75, 512, 0, 512, 3, 0),
    # one output-channel block (BN = Cout_pad = 128): odd tile counts (83 / 150 are not multiples of 8 / 16),
    # concatenated 64 + 64 input
    (8, 88, 160, 64, 0, 128, 3, 0), (8, 83, 150, 64, 64, 128, 3, 0), (6, 72, 160, 128, 0, 128, 3, 0),
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_tc_matches_torch(case):
    """wgmma implicit-GEMM conv + bias + LeakyReLU vs conv2d in float64 on the same fp16-rounded operands. Bar
    (tests/helpers.py): ulp16(ref) + 2^-16 * S for fp16 outputs, 2^-16 * S for the fp32 heads, S = conv2d(|x|, |w|) + |b|."""
    N, H, W, C1, C2, Cout, K, mode = case
    Lm, L = _lib()
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    x1 = torch.randn((N, C1, H, W), generator=g).to(DEV)
    x2 = torch.randn((N, C2, H, W), generator=g).to(DEV) if C2 else None
    w = (torch.randn((Cout, C1 + C2, K, K), generator=g) / np.sqrt((C1 + C2) * K * K)).to(DEV)
    b = (torch.randn((Cout,), generator=g) * 0.1).to(DEV)
    a1 = to_nhwc16(x1)
    a2 = to_nhwc16(x2) if C2 else None
    wp, Cp = pack_w(w, C1, C2)
    bp = torch.zeros(Cp, device=DEV)
    bp[:Cout] = b
    out = torch.full((N, H, W, Cp if mode == 0 else 8), float("nan"),
                     dtype=torch.float16 if mode == 0 else torch.float32, device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    Lm.check(L.v2e_conv2d_lrelu_sm100(p(a1), a1.shape[-1], p(a2), a2.shape[-1] if C2 else 0, p(wp), p(bp), Cp,
                                      K, K, N, H, W, p(out), Cp, mode, min(Cout, 8), ctypes.c_float(0.1), st))
    torch.cuda.synchronize()
    xin = torch.cat([x1, x2], 1) if C2 else x1
    ref, S = conv_ref64(xin.half(), w.half(), b, K // 2)
    ref, S = ref.permute(0, 2, 3, 1), S.permute(0, 2, 3, 1)
    co = min(Cout, out.shape[-1])
    r = err_ratio(out[..., :co], ref[..., :co], conv_bound(ref[..., :co], S[..., :co], fp16_out=mode == 0))
    assert r <= 1.0, r
    if mode == 0 and Cp > Cout:   # padded output channels must be exactly lrelu(0) = 0
        assert (out[..., Cout:] == 0).all()


STRIP_CASES = [
    # N, H, W, C1, C2, Cout, K, out_mode  (W >= 512: layers that run on the strip kernel)
    (1, 4, 512, 64, 0, 32, 3, 0), (1, 40, 512, 32, 0, 32, 3, 0), (1, 33, 530, 16, 0, 32, 3, 0),
    (1, 70, 512, 32, 0, 32, 7, 0), (2, 64, 640, 12, 0, 32, 7, 0), (2, 75, 576, 32, 32, 32, 3, 0),
    (1, 48, 640, 32, 0, 64, 5, 0), (1, 60, 512, 32, 0, 5, 3, 1), (3, 5, 513, 64, 0, 32, 3, 0),
    # output channels split over two CTA classes (weights of a slice resident), 2-slab inputs, short items
    (1, 37, 640, 64, 0, 64, 5, 0), (1, 20, 640, 128, 0, 64, 3, 0), (2, 24, 512, 64, 64, 64, 3, 0),
    (1, 2, 512, 32, 0, 32, 7, 0), (1, 1, 640, 16, 0, 32, 3, 0),
    # 346x260 network width (320 = 2.5 strips)
    (2, 30, 320, 32, 0, 32, 7, 0), (1, 17, 320, 32, 32, 32, 3, 0), (1, 9, 256, 32, 0, 5, 3, 1),
    # every CTA walks several items (132 SMs): ring counters and parities carried from item to item, the producer
    # filling the next item's rows while the consumers finish the current one.
    # 7x7, one CTA per SM: 10 strips x 8 segments x 8 images = 640 items on 132 CTAs
    (8, 176, 1280, 32, 0, 32, 7, 0),
    # 3x3, 16 channels, two CTAs per SM: 10 strips x 8 segments x 8 images = 640 items on 264 CTAs
    (8, 96, 1280, 16, 0, 32, 3, 0),
    # 5x5, 64 channels, output channels split over two CTA classes: 5 strips x 8 segments x 8 images = 320 items
    # on 66 CTAs per class
    (8, 88, 640, 64, 0, 64, 5, 0),
]


def pack_w_strip(w, C1, C2, KC):
    """fp16 [slabs][taps][Cout_pad][KC] (include/v2e_b200.h, v2e_conv2d_lrelu_sm100_strip)."""
    Cout, Cin, KH, KW = w.shape
    C1p, C2p = pad16(C1), (pad16(C2) if C2 else 0)
    Cp = cout_pad(Cout)
    full = torch.zeros((Cp, KH * KW, C1p + C2p), dtype=torch.float16, device=w.device)
    wt = w.permute(0, 2, 3, 1).reshape(Cout, KH * KW, Cin).half()
    full[:Cout, :, :C1] = wt[:, :, :C1]
    if C2:
        full[:Cout, :, C1p:C1p + C2] = wt[:, :, C1:]
    slabs = (C1p + C2p) // KC
    return full.reshape(Cp, KH * KW, slabs, KC).permute(2, 1, 0, 3).contiguous(), Cp


@pytest.mark.parametrize("case", STRIP_CASES)
def test_conv_strip_kernel_matches_torch(case):
    """Strip kernel (resident weights, input-row ring, descriptor-shifted taps, two warpgroups taking turns over
    pairs of output rows) vs conv2d in float64 on the same fp16-rounded operands. Same bar as the per-tap kernel."""
    N, H, W, C1, C2, Cout, K, mode = case
    Lm, L = _lib()
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    x1 = torch.randn((N, C1, H, W), generator=g).to(DEV)
    x2 = torch.randn((N, C2, H, W), generator=g).to(DEV) if C2 else None
    w = (torch.randn((Cout, C1 + C2, K, K), generator=g) / np.sqrt((C1 + C2) * K * K)).to(DEV)
    b = (torch.randn((Cout,), generator=g) * 0.1).to(DEV)
    a1 = to_nhwc16(x1)
    a2 = to_nhwc16(x2) if C2 else None
    Cp = cout_pad(Cout)
    KC = L.v2e_conv_strip_pick_kc(a1.shape[-1], a2.shape[-1] if C2 else 0, Cp, K, K, W)
    assert KC in (16, 32, 64), "case must qualify for the strip kernel"
    wp, Cp = pack_w_strip(w, C1, C2, KC)
    bp = torch.zeros(Cp, device=DEV)
    bp[:Cout] = b
    out = torch.full((N, H, W, Cp if mode == 0 else 8), float("nan"),
                     dtype=torch.float16 if mode == 0 else torch.float32, device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    Lm.check(L.v2e_conv2d_lrelu_sm100_strip(p(a1), a1.shape[-1], p(a2), a2.shape[-1] if C2 else 0, p(wp), p(bp), Cp,
                                            K, K, N, H, W, p(out), Cp, mode, min(Cout, 8), ctypes.c_float(0.1), st))
    torch.cuda.synchronize()
    xin = torch.cat([x1, x2], 1) if C2 else x1
    ref, S = conv_ref64(xin.half(), w.half(), b, K // 2)
    ref, S = ref.permute(0, 2, 3, 1), S.permute(0, 2, 3, 1)
    co = min(Cout, out.shape[-1])
    r = err_ratio(out[..., :co], ref[..., :co], conv_bound(ref[..., :co], S[..., :co], fp16_out=mode == 0))
    assert r <= 1.0, r


def test_full_resolution_unet_matches_float32_reference():
    """BASELINE resolution (1280x720 -> 1280x704 network): the layers that run on the strip kernel only
    exist at this width. One frame pair, flow UNet + one interpolated frame vs the float32 torch
    reference. Tolerances as in the small-size test."""
    from v2e_b200.slomo import SloMoEngine
    sd_fc, sd_at = _weights(5)
    H, W = 720, 1280
    frames = __import__("make_golden_slomo_frames").smooth_frames(2, H, W, 11, dx=6, dy=2, up=16)
    eng = SloMoEngine(sd_fc, sd_at, (W, H), 1, DEV)
    eng.set_pairs(torch.from_numpy(frames).to(DEV))
    flow = eng.flow_out().clone().cpu()[..., :4].permute(0, 3, 1, 2)
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    I, _ = slomo_ref.load_pair_tensors(frames, (eng.w, eng.h))
    ref_flow, ref_outs = slomo_ref.interp_batch(sd_fc, sd_at, I[:1], I[1:2], 1)
    rms = ref_flow.pow(2).mean().sqrt().item()
    assert (flow - ref_flow).abs().max().item() < 0.02 * rms + 0.02, ((flow - ref_flow).abs().max().item(), rms)
    out = torch.empty((1, H, W), dtype=torch.uint8, device=DEV)
    ft = torch.empty((1, eng.h, eng.w), dtype=torch.float32, device=DEV)
    eng.interp(0.5, out, ft)
    d = (ft.cpu() - ref_outs[0][1][:, 0]).abs()
    assert d.max().item() < 0.01 and d.mean().item() < 0.001, (d.max().item(), d.mean().item())
    eng.close()


@pytest.mark.parametrize("sizes", [((346, 260), (320, 256), 1), ((320, 256), (346, 260), 0),
                                   ((1280, 720), (1280, 704), 1), ((1280, 704), (1280, 720), 0),
                                   ((100, 70), (96, 64), 1), ((96, 64), (100, 70), 0), ((130, 96), (128, 96), 1)])
def test_resize_is_pillow_exact(sizes):
    """8-bit LANCZOS / BILINEAR resampling must equal Pillow bit for bit (dataloader.py:142, slomo.py:438)."""
    from PIL import Image
    (sw, sh), (dw, dh), filt = sizes
    Lm, L = _lib()
    rng = np.random.default_rng(sw * 7 + dh)
    imgs = rng.integers(0, 256, (3, sh, sw), dtype=np.uint8)
    imgs[1] = np.kron(rng.integers(0, 256, (sh // 4 + 1, sw // 4 + 1), dtype=np.uint8), np.ones((4, 4), np.uint8))[:sh, :sw]
    r = ctypes.c_void_p()
    Lm.check(L.v2e_resize_create(sw, sh, dw, dh, filt, 3, ctypes.byref(r)))
    src = torch.from_numpy(imgs).to(DEV)
    dst = torch.zeros((3, dh, dw), dtype=torch.uint8, device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    Lm.check(L.v2e_resize_run(r, ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr()), 3, st))
    got = dst.cpu().numpy()
    L.v2e_resize_destroy(r)
    for i in range(3):
        want = np.asarray(Image.fromarray(imgs[i]).resize((dw, dh), Image.LANCZOS if filt else Image.BILINEAR))
        assert np.array_equal(got[i], want), "image %d: %d pixels differ" % (i, int((got[i] != want).sum()))


def _weights(seed):
    return (slomo_ref.make_test_weights(100 + seed, 2, 4, head_gain=25.0),
            slomo_ref.make_test_weights(200 + seed, 12, 5, head_gain=0.3))


def test_unets_and_blend_match_float32_reference():
    """Flow UNet, interpolation UNet and the blended frame vs the float32 torch reference on the same
    inputs. Tolerances (fp16 operands through 23 layers): network outputs within 2% of their RMS
    (max error) ; blended frame Ft_p within 0.01 (2.5 DN) max, 0.001 (0.25 DN) mean."""
    from v2e_b200.slomo import SloMoEngine
    sd_fc, sd_at = _weights(3)
    H, W, B = 96, 128, 2
    frames = np.stack([np.asarray(f) for f in __import__("make_golden_slomo_frames").smooth_frames(B + 1, H, W, 5)])
    eng = SloMoEngine(sd_fc, sd_at, (W, H), B, DEV)
    fr = torch.from_numpy(frames).to(DEV)
    eng.set_pairs(fr)
    flow = eng.flow_out().clone().cpu()[..., :4].permute(0, 3, 1, 2)
    I, _ = slomo_ref.load_pair_tensors(frames, (W, H))
    ref_flow, ref_outs = slomo_ref.interp_batch(sd_fc, sd_at, I[:B], I[1:B + 1], 2)
    rms = ref_flow.pow(2).mean().sqrt().item()
    assert (flow - ref_flow).abs().max().item() < 0.02 * rms + 0.02, ((flow - ref_flow).abs().max().item(), rms)
    out = torch.empty((B, H, W), dtype=torch.uint8, device=DEV)
    ft = torch.empty((B, H, W), dtype=torch.float32, device=DEV)
    for k in range(2):
        eng.interp((k + 0.5) / 2, out, ft)
        ref_intrp, ref_ft = ref_outs[k]
        d = (ft.cpu() - ref_ft[:, 0]).abs()
        assert d.max().item() < 0.01 and d.mean().item() < 0.001, (d.max().item(), d.mean().item())
        q = out.cpu().numpy().astype(np.int32) - slomo_ref.to_u8(ref_ft)[:, 0].numpy().astype(np.int32)
        assert np.abs(q).max() <= 3 and np.abs(q).mean() < 0.3
    eng.close()


@pytest.mark.parametrize("name", ["slomo_64x96_u2_b1", "slomo_70x100_u3_b2", "slomo_96x130_auto"])
def test_superslomo_dropin_matches_reference_golden(name, tmp_path):
    """SuperSloMo.interpolate (folder of .npy in, .png out) against the frames the unmodified reference
    wrote for the same inputs and weights. Same frame count, same interpTimes (exact), uint8 frames
    within 3 DN max / 0.3 DN mean (fp16 tensor-core convolutions vs the reference's fp32 CPU convs)."""
    import cv2
    from v2e_b200.slomo import SuperSloMo
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    seed = int(z["seed"])
    sd_fc, sd_at = _weights(seed)
    import hashlib
    dig = "".join(hashlib.sha1(b"".join(sd[k].numpy().tobytes() for k in sorted(sd))).hexdigest() for sd in (sd_fc, sd_at))
    if dig != str(z["weights_sha1"]):
        pytest.skip("torch.randn on this host does not reproduce the fixture's weights")
    src, dst = tmp_path / "src", tmp_path / "dst"
    src.mkdir(); dst.mkdir()
    for i, f in enumerate(z["frames"]):
        np.save(str(src / ("%08d.npy" % i)), f)
    s = SuperSloMo(model=None, auto_upsample=bool(z["auto"]), upsampling_factor=int(z["U"]),
                   batch_size=int(z["batch_size"]), state_dicts={"state_dictFC": sd_fc, "state_dictAT": sd_at})
    H, W = z["frames"].shape[1:]
    times, avg = s.interpolate(str(src), str(dst), (W, H))
    n = len(os.listdir(str(dst)))
    got = np.stack([cv2.imread(str(dst / ("%d.png" % i)), cv2.IMREAD_GRAYSCALE) for i in range(n)])
    assert got.shape == z["out"].shape
    assert np.array_equal(times, z["times"]) and avg == float(z["avg"])
    d = np.abs(got.astype(np.int32) - z["out"].astype(np.int32))
    assert d.max() <= 3 and d.mean() < 0.3, (d.max(), d.mean())
    s.cleanup()


def test_superslomo_errors():
    from v2e_b200.slomo import SuperSloMo
    with pytest.raises(ValueError):
        SuperSloMo(model=None, auto_upsample=False, upsampling_factor=1)
    s = SuperSloMo(model="/nonexistent.ckpt", auto_upsample=False, upsampling_factor=2)
    with pytest.raises(FileNotFoundError):
        s.interpolate_frames(np.zeros((3, 64, 64), np.uint8))
    with pytest.raises(ValueError):
        s.interpolate("/tmp", None, (64, 64))


def _clip_sharded_worker(rank, world, port, frames, kw, q):
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)     # gloo moves CUDA tensors through the host:
    try:                                                              # two ranks can share the one test GPU
        from v2e_b200 import EventEmulator, SuperSloMo, V2EPipeline
        fc, at = _weights(5)
        sl = SuperSloMo(model=None, auto_upsample=False, upsampling_factor=3, batch_size=2,
                        state_dicts={'state_dictFC': fc, 'state_dictAT': at})
        em = EventEmulator(device="cuda:0", seed=9, shard=(rank, world, None), **kw)
        rows, t, nf = V2EPipeline(sl, em).run_clip_sharded(frames, 0.2)
        q.put((rank, rows, nf))
        sl.cleanup()
    finally:
        dist.destroy_process_group()


def test_one_clip_sharded_over_two_ranks_matches_single_gpu():
    """BASELINE config 5 layout: SloMo sharded over frame pairs, all-to-all of uint8 row bands, pixel model
    sharded over rows with the per-frame all-reduce(MAX). The union of the two ranks' events must equal the
    single-process pipeline's events frame by frame (noise off: no per-frame draws; thresholds seeded)."""
    import socket
    import torch.multiprocessing as mp
    from v2e_b200 import EventEmulator, SuperSloMo, V2EPipeline
    rng = np.random.default_rng(4)
    big = np.kron(rng.integers(30, 220, (14, 30)).astype(np.uint8), np.ones((8, 8), np.uint8))
    frames = np.stack([big[3:3 + 96, 4 * k:4 * k + 128] for k in range(6)])     # 5 pairs, 96x128
    kw = dict(cutoff_hz=200, leak_rate_hz=0, shot_noise_rate_hz=0, refractory_period_s=0.001, sigma_thres=0.02)
    fc, at = _weights(5)
    sl = SuperSloMo(model=None, auto_upsample=False, upsampling_factor=3, batch_size=2,
                    state_dicts={'state_dictFC': fc, 'state_dictAT': at})
    em = EventEmulator(device="cuda:0", seed=9, rng_mode="device", **kw)
    ev, offs, t, nf = V2EPipeline(sl, em).run(frames, 0.2)
    sl.cleanup()
    assert nf == 15 and ev.shape[0] > 0
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_clip_sharded_worker, args=(r, 2, port, frames, kw, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(r[2] == 15 for r in res)
    got = np.concatenate([r[1] for r in sorted(res, key=lambda r: r[0])], 0)
    assert got.shape == ev.shape
    key = lambda e: e[np.lexsort((e[:, 3], e[:, 1], e[:, 2], e[:, 0]))]
    assert np.array_equal(key(got), key(np.asarray(ev)))


@pytest.mark.parametrize("case", [(2, 48, 640, 64, 32), (1, 38, 512, 64, 17), (1, 8, 768, 64, 32)])
def test_fused_upsample_conv_matches_torch(case):
    """conv3x3(bilinear_up2(x)) + bias + LeakyReLU with the up-sampling folded into the filter (strip2up + frame
    kernel) vs interpolate -> conv2d in float64 on the same fp16-rounded input and weights. The folded filter is
    rounded to fp16 after the combination (relative error 2^-11 per folded weight) and the frame kernel rounds each
    bilinear sample to fp16: bar ulp16(ref) + 2^-10 * S', S' = conv2d(interpolate(|x|), |w|) + |b|, on the interior
    and on the 2-pixel frame alike."""
    N, H, W, C, Cout = case                       # H, W: output size
    Lm, L = _lib()
    assert L.v2e_conv_up2_supported_c(C, cout_pad(Cout), W) == 1
    g = torch.Generator().manual_seed(hash(case) & 0xFFFF)
    x = torch.randn((N, C, H // 2, W // 2), generator=g).to(DEV)
    w = (torch.randn((Cout, C, 3, 3), generator=g) / np.sqrt(C * 9)).to(DEV)
    b = (torch.randn((Cout,), generator=g) * 0.1).to(DEV)
    a = to_nhwc16(x)
    Cp = cout_pad(Cout)
    wp, _ = pack_w(w, C, 0)
    fold = np.zeros(((C // 64) * 2 * 3 * 6 * Cp * 64,), np.float16)
    wh = np.ascontiguousarray(w.half().float().cpu().numpy())
    Lm.check(L.v2e_conv_up2_fold_weights(wh.ctypes.data_as(ctypes.c_void_p), Cout, C, Cp, C,
                                         fold.ctypes.data_as(ctypes.c_void_p)))
    fold_d = torch.from_numpy(fold).to(DEV)
    bp = torch.zeros(Cp, device=DEV)
    bp[:Cout] = b
    out = torch.full((N, H, W, Cp), float("nan"), dtype=torch.float16, device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    Lm.check(L.v2e_conv2d_up2_lrelu_sm100(p(a), C, p(fold_d), p(wp), p(bp), Cp, N, H, W, p(out), Cp, ctypes.c_float(0.1), st))
    torch.cuda.synchronize()
    up2 = lambda t: torch.nn.functional.interpolate(t, scale_factor=2, mode="bilinear", align_corners=False)
    x16 = x.half().double()
    ref, _ = conv_ref64(up2(x16), w.half(), b, 1)
    _, S = conv_ref64(up2(x16.abs()), w.half(), b, 1)
    bar = conv_bound(ref, S, acc=2.0 ** -10)
    got = out[..., :Cout].permute(0, 3, 1, 2)
    assert torch.isfinite(out.float()).all()
    frame = torch.ones_like(ref, dtype=torch.bool)
    frame[..., 2:-2, 2:-2] = False
    r = (got.double() - ref).abs() / bar
    assert r[~frame].max().item() <= 1.0 and r[frame].max().item() <= 1.0, (r[~frame].max().item(), r[frame].max().item())
    if Cp > Cout:
        assert (out[..., Cout:] == 0).all()


def test_fused_average_pool_is_bit_identical_to_the_separate_kernel():
    """The 2x2 average pools after conv2 (and down1.conv2 on wide frames) ride in the strip kernel's epilogue.
    The mean of four fp16 values in float32 is exact whatever the order, so the network heads must not change by
    one bit when the fusion is switched off (v2e_slomo_set_option(h, 2, 1))."""
    from v2e_b200.slomo import SloMoEngine
    sd_fc, sd_at = _weights(7)
    for (W, H) in ((1280, 96), (346, 260)):
        frames = __import__("make_golden_slomo_frames").smooth_frames(3, H, W, 5, dx=4, dy=1, up=16)
        eng = SloMoEngine(sd_fc, sd_at, (W, H), 2, DEV)
        fr = torch.from_numpy(frames).to(DEV)
        outs = []
        for off in (0, 1):
            _lib()[0].check(eng.lib.v2e_slomo_set_option(eng._h, 2, off))
            eng.set_pairs(fr)
            flow = eng.flow_out().clone()
            out = torch.empty((2, H, W), dtype=torch.uint8, device=DEV)
            ft = torch.empty((2, eng.h, eng.w), dtype=torch.float32, device=DEV)
            eng.interp(0.3, out, ft)
            outs.append((flow, ft.clone(), out.clone()))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2])
        eng.close()


def _scaled(sd, first, last, names=("conv1", "conv3")):
    out = {k: v.clone() for k, v in sd.items()}
    out[names[0] + ".weight"] *= first
    out[names[0] + ".bias"] *= first
    out[names[1] + ".weight"] *= last
    return out


def test_fp16_dynamic_range_large_activations_still_match_float32():
    """The reference computes in float32 (TF32 multiplies on Ampere+); here operands are fp16 (same 10-bit mantissa,
    5-bit exponent). Weights scaled so that every hidden activation is ~400x larger (thousands, where fp16's absolute
    spacing is 2-8) with the head scaled back: LeakyReLU networks are positively homogeneous, so the float32 result
    is the unscaled one and the fp16 path must still match it to the usual tolerance -- relative precision, not
    absolute, is what the layers need. Biases of the hidden layers are scaled consistently by the first layer only,
    so this is not an exact rescaling: the comparison is against the float32 reference of the SAME scaled weights."""
    from v2e_b200.slomo import SloMoEngine
    sd_fc, sd_at = _weights(3)
    sd_fc, sd_at = _scaled(sd_fc, 400.0, 1 / 400.0), _scaled(sd_at, 400.0, 1 / 400.0)
    H, W, B = 96, 128, 2
    frames = np.stack([np.asarray(f) for f in __import__("make_golden_slomo_frames").smooth_frames(B + 1, H, W, 5)])
    eng = SloMoEngine(sd_fc, sd_at, (W, H), B, DEV)
    eng.set_pairs(torch.from_numpy(frames).to(DEV))
    flow = eng.flow_out().clone().cpu()[..., :4].permute(0, 3, 1, 2)
    I, _ = slomo_ref.load_pair_tensors(frames, (W, H))
    ref_flow, ref_outs = slomo_ref.interp_batch(sd_fc, sd_at, I[:B], I[1:B + 1], 2)
    rms = ref_flow.pow(2).mean().sqrt().item()
    assert torch.isfinite(flow).all()
    assert (flow - ref_flow).abs().max().item() < 0.03 * rms + 0.03, ((flow - ref_flow).abs().max().item(), rms)
    out = torch.empty((B, H, W), dtype=torch.uint8, device=DEV)
    ft = torch.empty((B, H, W), dtype=torch.float32, device=DEV)
    for k in range(2):
        eng.interp((k + 0.5) / 2, out, ft)
        d = (ft.cpu() - ref_outs[k][1][:, 0]).abs()
        assert d.max().item() < 0.02 and d.mean().item() < 0.002, (d.max().item(), d.mean().item())
    eng.check_finite()
    eng.close()


def test_fp16_overflow_fails_loudly():
    """Activations beyond fp16's 65504 become inf / nan in the heads: the drop-in must raise, not return garbage frames."""
    from v2e_b200 import SuperSloMo
    sd_fc, sd_at = _weights(3)
    sd_at = _scaled(sd_at, 3.0e5, 1.0)
    frames = np.stack([np.asarray(f) for f in __import__("make_golden_slomo_frames").smooth_frames(3, 96, 128, 5)])
    sl = SuperSloMo(model=None, auto_upsample=False, upsampling_factor=2, batch_size=2,
                    state_dicts={'state_dictFC': sd_fc, 'state_dictAT': sd_at})
    with pytest.raises(FloatingPointError):
        sl.interpolate_frames(frames)
    sl.cleanup()


def test_end_to_end_event_delta_of_the_fp16_slomo():
    """SURVEY.md 8(d) parity criterion for the reduced-precision SloMo: "report max / mean abs diff of the uint8 frames
    and the induced event-count delta". Same source frames (scripts/gradients.py's moving bump, 346x260, x10) through
    the fp16 tensor-core SloMo and through the float32 restatement of the reference; both frame sets through the same
    pixel model with noise off. Bars: frames within 3 DN (observed 1), events within 1 % in total and per polarity."""
    import bench
    d = bench.slomo_event_delta(DEV, bench.slomo_weights())
    assert d["dn_max"] <= 3 and d["dn_mean"] < 0.3, d
    assert d["events_fp32"] > 10000
    assert abs(d["delta_events"]) <= 0.01 * d["events_fp32"], d
    assert abs(d["delta_on"]) <= 0.01 * d["events_fp32"] and abs(d["delta_off"]) <= 0.01 * d["events_fp32"], d
