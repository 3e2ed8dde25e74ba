"""Weight gradient of the 8-channel discriminator stems (5x5, 8 -> 64 channels, models/gan.py:163-166) from the RAW input:
b3d_conv2d_wgrad_tf32 with fold_kh > 0 (kernel wgrad_stem) against an fp64 reference of the folded layer's gradient,
dW'[s][co][r*8 + ci] = sum dY[n,y,x,co] * X[n, y + r - pad_y, x + s, ci], in both dW layouts, with a dY row pitch and at
the edges of its K slicing (a width that is not a multiple of 32, one image).  Tolerance 4e-3 of the largest magnitude, the
tf32 class of tests/test_bench_shapes_gpu.py.  Then one banked discriminator step at cfg3 through GANTrainer: the stem's
weight gradient runs on the raw input (no folded tensor is kept for the backward) and the step lands where the materialised
fold lands, within the run-to-run band of the split-K atomics."""
import ctypes
import sys

import pytest
import torch

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import gan_common as GC                  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 4e-3
DEV = "cuda:0"
KH = KW = 5
CF = 64                                  # folded channels: 8 * KH real, the rest zero


def _ref(dy, x, pad_y):
    """fp64 [KW][Cout][CF] gradient of the folded layer."""
    N, Hout, Wout, Cout = dy.shape
    xp = torch.nn.functional.pad(x.double(), (0, 0, 0, 0, pad_y, pad_y))
    d = dy.double().reshape(-1, Cout).t()
    out = torch.zeros(KW, Cout, CF, dtype=torch.float64, device=dy.device)
    for r in range(KH):
        for s in range(KW):
            out[s, :, 8 * r:8 * r + 8] = d @ xp[:, r:r + Hout, s:s + Wout].reshape(-1, 8)
    return out


# N, H, W (x-padded raw input), Cout, pad_y, dY row pitch (0: dense)
CASES = [
    ("cfg3", 64, 256, 260, 64, 2, 0),                # D1.conv1 of cfg3's D step (2B = 64 images at 256^2)
    ("cfg5_d3", 16, 128, 132, 64, 2, 0),             # cfg5's third discriminator (2B = 16 images at 128^2)
    ("wout100", 3, 20, 104, 64, 2, 0),               # Wout = 100: the last 32-pixel segment of a row is partial
    ("n1", 1, 37, 68, 128, 2, 0),                    # one image, two 64-channel tiles
    ("pitch", 4, 48, 132, 64, 2, 133),               # dY read through a row pitch wider than Wout
]


@pytest.mark.parametrize("name,N,H,W,Cout,pad_y,pitch", CASES, ids=[c[0] for c in CASES])
def test_stem_wgrad_from_raw_input(name, N, H, W, Cout, pad_y, pitch):
    from b3d import check, last_variant, lib, ptr, stream_ptr
    Hout, Wout = H + 2 * pad_y - KH + 1, W - KW + 1
    g = torch.Generator(device=DEV).manual_seed(N * 31 + W)
    x = torch.randn(N, H, W, 8, device=DEV, generator=g)
    dyw = torch.randn(N, Hout, pitch or Wout, Cout, device=DEV, generator=g)
    dy = dyw[:, :, :Wout]
    ref = _ref(dy, x, pad_y)
    scale = float(ref.abs().max())
    st = stream_ptr(x)

    tm = torch.zeros(KW, Cout, CF, device=DEV)                          # the bank's tap-major sink
    check(lib.b3d_conv2d_wgrad_tf32(ctypes.c_void_p(dyw.data_ptr()), ptr(x), ptr(tm), N, H, W, CF, Hout, Wout, Cout, 1, KW,
                                    pad_y, 1, 0, 1, KH, pitch, st))
    assert last_variant().startswith("wgrad_stem<"), last_variant()
    dense = torch.zeros(Cout, CF, 1, KW, device=DEV)
    check(lib.b3d_conv2d_wgrad_tf32(ctypes.c_void_p(dyw.data_ptr()), ptr(x), ptr(dense), N, H, W, CF, Hout, Wout, Cout, 1, KW,
                                    pad_y, 1, 0, 0, KH, pitch, st))
    torch.cuda.synchronize()
    err_tm = float((tm.double() - ref).abs().max())
    err_dense = float((dense[:, :, 0].permute(2, 0, 1).double() - ref).abs().max())
    assert err_tm <= TOL * scale, (name, "tap-major", err_tm, scale)
    assert err_dense <= TOL * scale, (name, "[Cout][Cin][1][kw]", err_dense, scale)
    assert torch.equal(tm[:, :, 8 * KH:], torch.zeros_like(tm[:, :, 8 * KH:]))
    assert torch.equal(dense[:, 8 * KH:], torch.zeros_like(dense[:, 8 * KH:]))


def test_stem_wgrad_rejects_unsupported_geometry():
    from b3d import lib, ptr, stream_ptr
    x = torch.randn(1, 16, 36, 8, device=DEV)
    dy = torch.randn(1, 16, 32, 64, device=DEV)
    dw = torch.zeros(KW, 64, CF, device=DEV)
    # three folded rows do not fill 64 channels; stride 2 is not a stem
    assert lib.b3d_conv2d_wgrad_tf32(ptr(dy), ptr(x), ptr(dw), 1, 16, 36, CF, 16, 32, 64, 1, KW, 1, 1, 0, 1, 3, 0, stream_ptr(x)) != 0
    assert lib.b3d_conv2d_wgrad_tf32(ptr(dy), ptr(x), ptr(dw), 1, 16, 36, CF, 16, 32, 64, 1, KW, 2, 2, 0, 1, KH, 0, stream_ptr(x)) != 0


# ------------------------------------------------------------------------------------------------ one banked D step at cfg3
def _old_banked(x_nchw, lw, pad_y=0, stride=1, leaky=1.0, pad_out=0, pad_mode=1, x_crop=0, stats=None, link_in=None,
                link_out=None):
    """The stems on the materialised fold (b3d.ew.fold_rows + the generic weight-gradient kernel): the path D steps took
    before the raw-input weight gradient."""
    import b3d.conv as C
    from b3d.ew import fold_rows
    if not lw.fold:
        return C.conv2d_banked(x_nchw, lw, pad_y, stride, leaky, pad_out, pad_mode, x_crop, stats, link_in, link_out)
    x = fold_rows(x_nchw.permute(0, 2, 3, 1), lw.kh, pad_y, lw.Cinp)
    y = C._Conv.apply(x, lw.wf, lw.bias, lw, int(pad_y), int(stride), float(leaky), int(pad_out), int(pad_mode), int(x_crop),
                      stats, 0, link_in, link_out)
    return y.permute(0, 3, 1, 2)


def _d_step(batch, old):
    import bench
    import b3d.conv as C
    import models.gan as MG
    from gan_training import GANTrainer
    torch.manual_seed(11)
    tr = GANTrainer(bench.gan_args(256, 2), mesh_template=None, device=DEV)
    C.VARIANT_LOG = []
    if old:
        MG.conv2d_banked = _old_banked
    try:
        loss = float(tr.d_step(batch["X_tex"], batch["X_alpha"], batch["X_mesh"], batch["C"], batch["noise"]))
        torch.cuda.synchronize()
        launched = list(C.VARIANT_LOG)
    finally:
        C.VARIANT_LOG, MG.conv2d_banked = None, C.conv2d_banked
    params = {n: p.detach().clone() for n, p in tr.trainer.discriminator.named_parameters()}
    del tr
    torch.cuda.empty_cache()
    return loss, params, launched


def test_banked_d_step_uses_the_raw_input_stem():
    args = GC.make_args(256, 2)
    z, c, alpha, tex, mesh = GC.inputs(args, B=32, seed=21)
    batch = dict(X_tex=tex.to(DEV), X_alpha=alpha.to(DEV), X_mesh=mesh.to(DEV), C=c.to(DEV), noise=z.to(DEV))
    l_new, p_new, launched = _d_step(batch, old=False)
    l_old, p_old, launched_old = _d_step(batch, old=True)
    l_old2, p_old2, _ = _d_step(batch, old=True)
    # d1's 8-channel stem moves from the generic kernel on the folded tensor to the raw-input kernel; d2's 11-channel mesh
    # stem stays on the folded tensor
    generic = "wgrad_wgmma<64,4,4,1>"
    assert launched.count("wgrad_stem<5,4,3>") == 1 and "wgrad_stem<5,4,3>" not in launched_old, (launched, launched_old)
    assert launched.count(generic) == launched_old.count(generic) - 1 >= 1, (launched, launched_old)
    # split-K atomics sum in a different order from run to run, and Adam's first step turns a gradient that cancels to ~0
    # into a full +-lr step either way: the new path must stay within 4x the spread of two runs of the old one
    band = max(float((p_old2[n] - p).abs().max()) for n, p in p_old.items())
    diff = max(float((p_new[n] - p).abs().max()) for n, p in p_old.items())
    print("D step: loss new / old / old again", l_new, l_old, l_old2, "largest parameter difference new", diff, "band", band)
    assert abs(l_new - l_old) <= 4 * abs(l_old2 - l_old) + 1e-5 * abs(l_old)
    assert diff <= 4 * band + 1e-6, (diff, band)
