"""The 64-output-channel tiles of the wgmma convolution (conv_wgmma<64,8> and the conv_wgmma_rowwin<64,KW,S> row windows):
weights as the wgmma M operand, 128-pixel tiles as the N operand, one work item per consumer warpgroup.

Every 64-channel geometry cfg3 dispatches, at batch 32 and 64, forward and input gradient, against an fp64 convolution
of two images of the batch (images are independent); epilogue statistics against the sums of the stored output (the bounds
of test_bench_shapes_gpu.py::test_epilogue_statistics).  Also the epilogue's edges: the fused LeakyReLU adjoint (mask),
sums-only statistics, a pitched dY, the four merged parity classes, strip launches (widths 130 and 129), pad_out, x_crop,
CTAs with an odd number of items (one consumer warpgroup takes one more than the other) and grids with fewer items than
SMs."""
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 4e-3
DEV = "cuda:0"
SEEN = set()
REF_IMGS = (0, -1)          # images of the batch compared against the fp64 reference


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _log(fn):
    import b3d.conv as C
    C.VARIANT_LOG = []
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        SEEN.update(C.VARIANT_LOG)
        C.VARIANT_LOG = None
    return out


def _close(a, r, what):
    assert a.shape == r.shape, (what, tuple(a.shape), tuple(r.shape))
    err, ref = float((a.double() - r).abs().max()), float(r.abs().max())
    assert err <= TOL * ref, (what, err, ref)


def _check_stats(stats, y, C, sums_only=False):
    """fp64 per-channel sums (and sums of squares) accumulated by the epilogue == those of the stored tensor y (NHWC)."""
    yd = y.double().reshape(-1, y.shape[-1])[:, :C]
    s, q = yd.sum(0), (yd * yd).sum(0)
    assert float((stats[:C] - s).abs().max()) <= 2e-6 * float(yd.abs().sum(0).max())
    if sums_only:
        assert float(stats[C:].abs().max()) == 0.0
    else:
        assert float((stats[C:2 * C] - q).abs().max()) <= 2e-6 * float(q.max())


def _sub(t):
    return t[list(REF_IMGS)]


def _ref_fwd(x, w, bias, pad_y, stride, x_crop=0):
    """fp64 forward of the reference images: x NHWC, w [Cout,Cin,kh,kw] -> NHWC."""
    xs = _sub(x).permute(0, 3, 1, 2).double()
    if x_crop:
        xs = xs[..., x_crop:xs.shape[3] - x_crop]
    y = torch.nn.functional.conv2d(xs, w.double(), bias.double() if bias is not None else None, stride=stride, padding=(pad_y, 0))
    return y.permute(0, 2, 3, 1)


def _ref_dgrad(gy, w, in_hw, pad_y, stride, x_crop=0):
    """fp64 input gradient of the reference images: gy NHWC, w [Cout,Cin,kh,kw] -> NHWC [n, H, W, Cin]."""
    H, W = in_hw
    g = _sub(gy).permute(0, 3, 1, 2).double()
    gx = torch.nn.grad.conv2d_input((g.shape[0], w.shape[1], H, W - 2 * x_crop), w.double(), g, stride=stride, padding=(pad_y, 0))
    return torch.nn.functional.pad(gx, (x_crop, x_crop)).permute(0, 2, 3, 1)


def _operands(N, Cin, H, W, Cout, k, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, Cin, generator=g).to(DEV)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).to(DEV)
    return x, w


# name, Cin, H, W (x-padded input), Cout, k, pad_y, stride, x_crop — the 64-output-channel forward launches of cfg3
FWD = [("G.blk6.conv1", 128, 256, 130, 64, 3, 1, 1, 0),          # conv_wgmma_rowwin<64,3,4>
       ("G.blk6.conv2", 64, 256, 130, 64, 3, 1, 1, 0),           # conv_wgmma_rowwin<64,3,4>
       ("G.blk6.short", 128, 256, 130, 64, 1, 0, 1, 1),          # conv_wgmma<64,8>, x_crop
       ("G.blk3_mesh.conv1", 256, 32, 18, 64, 3, 1, 1, 0)]       # conv_wgmma<64,8>, several rows per tile


@pytest.mark.parametrize("N", [32, 64])
@pytest.mark.parametrize("stats", [False, True])
@pytest.mark.parametrize("name,Cin,H,W,Cout,k,pad_y,stride,x_crop", FWD, ids=[c[0] for c in FWD])
def test_forward(name, Cin, H, W, Cout, k, pad_y, stride, x_crop, N, stats):
    import b3d.conv as C
    x, w = _operands(N, Cin, H, W, Cout, k, sum(map(ord, name)) + N)
    st = torch.zeros(2 * Cout, device=DEV, dtype=torch.float64) if stats else None
    y = _log(lambda: C._fprop(x, C.taps_layout(w), None, k, k, pad_y, stride, x_crop=x_crop, stats=st))
    _close(_sub(y), _ref_fwd(x, w, None, pad_y, stride, x_crop), name)
    if stats:
        _check_stats(st, y, Cout)


@pytest.mark.parametrize("N,W,pad_out", [(32, 130, 1), (64, 132, 2)])
def test_forward_bias_leaky_pad_out(N, W, pad_out):
    """bias + LeakyReLU in the epilogue, written into the interior of an x-padded buffer (main + 2-column strip launch)."""
    import b3d.conv as C
    x, w = _operands(N, 64, 64, W, 64, 3, W + pad_out)
    b = torch.randn(64, generator=torch.Generator().manual_seed(1)).to(DEV)
    y = _log(lambda: C._fprop(x, C.taps_layout(w), b, 3, 3, 1, 1, leaky=0.2, pad_out=pad_out))
    r = _ref_fwd(x, w, b, 1, 1)
    _close(_sub(y)[:, :, pad_out:y.shape[2] - pad_out], torch.where(r >= 0, r, 0.2 * r), "bias/leaky/pad_out")


@pytest.mark.parametrize("N", [32, 64])
@pytest.mark.parametrize("on_the_fly", [False, True])
def test_stem_forward(N, on_the_fly):
    """Discriminator stem, 5 rows of the raw 8-channel input folded into 64 channels: fold_rows + 1x5 row window
    (conv_wgmma_rowwin<64,5,3>) and the fold on the fly (conv_wgmma<64,8>, 32-byte-swizzled pixel tiles)."""
    import b3d.conv as C
    from b3d.ew import fold_rows
    g = torch.Generator().manual_seed(N + on_the_fly)
    xr = torch.randn(N, 64, 260, 8, generator=g).to(DEV)
    wf = torch.randn(5, 64, 64, generator=g) * 0.05
    wf[:, :, 40:] = 0
    wf = wf.to(DEV)
    st = torch.zeros(128, device=DEV, dtype=torch.float64)
    if on_the_fly:
        y = _log(lambda: C._fprop(xr, wf, None, 1, 5, stats=st, fold_kh=5, fold_pad=2))
    else:
        y = _log(lambda: C._fprop(fold_rows(xr, 5, 2, 64), wf, None, 1, 5, stats=st))
    w = wf[:, :, :40].reshape(5, 64, 5, 8).permute(1, 3, 2, 0)              # [s][co][r*8 + ci] -> [co][ci][r][s]
    _close(_sub(y), _ref_fwd(xr, w, None, 2, 1), "stem")
    _check_stats(st, y, 64)


def _mask_like(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(DEV)


@pytest.mark.parametrize("N", [32, 64])
@pytest.mark.parametrize("name,Cin,H,W,Cout,k,pad_y,stride,x_crop,masked,pitched", [
    ("G.blk6.conv2", 64, 256, 130, 64, 3, 1, 1, 0, True, True),       # rowwin<64,3,4>: width 130 = main + strip launch
    ("G.blk6.short", 64, 256, 130, 64, 1, 0, 1, 1, False, False),     # conv_wgmma<64,8>: x_crop
    ("D1.conv2", 64, 128, 130, 128, 4, 1, 2, 0, True, False),         # rowwin<64,2,5>: four merged parity classes, width 65
    ("D1.conv2.wide", 64, 64, 258, 128, 4, 1, 2, 0, True, False),     # parity classes of width 129: main + 1-column strip
    ("G.conv_final", 64, 64, 132, 32, 5, 2, 1, 0, False, False),      # rowwin<64,5,3>
])
def test_input_gradient(name, Cin, H, W, Cout, k, pad_y, stride, x_crop, masked, pitched, N):
    """Input gradient with 64 output channels (= the layer's input channels): the mask (LeakyReLU adjoint of the input's
    activation, slope 0.2) and the sums-only statistics of the fused adjoint, dY read in place from a padded buffer."""
    import b3d.conv as C
    if "conv_final" in name:
        N = N // 4          # the largest geometry; the tile / strip structure does not depend on the batch
    x, w = _operands(1, Cin, H, W, Cout, k, sum(map(ord, name)) + N)
    wf = w.permute(2, 3, 0, 1).reshape(k * k, Cout, Cin)
    Hout, Wout = (H + 2 * pad_y - k) // stride + 1, (W - 2 * x_crop - k) // stride + 1
    g = torch.Generator().manual_seed(7 + N)
    if pitched:
        gbuf = torch.randn(N, Hout, Wout + 2, Cout, generator=g).to(DEV)
        gy = gbuf[:, :, 1:Wout + 1]
    else:
        gy = torch.randn(N, Hout, Wout, Cout, generator=g).to(DEV)
    mask = _mask_like((N, H, W, Cin), 11) if masked else None
    sums = torch.zeros(2 * Cin, device=DEV, dtype=torch.float64) if masked else None
    gx = _log(lambda: C._dgrad(gy, C._d_layout(wf), (H, W), k, k, pad_y, stride, x_crop, g_pitch=(Wout + 2) if pitched else 0,
                               mask=mask, slope=0.2, sums=sums))
    r = _ref_dgrad(gy, w, (H, W), pad_y, stride, x_crop)
    if masked:
        r = r * torch.where(_sub(mask) >= 0, 1.0, 0.2).double()
    _close(_sub(gx), r, name)
    if masked:
        _check_stats(sums, gx, Cin, sums_only=True)


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("items", ["odd_per_cta", "fewer_than_sms"])
def test_work_distribution(items, k):
    """Items alternate between the two consumer warpgroups of a CTA: three items per CTA (warpgroup 0 takes two), and a
    grid of fewer items than SMs (CTAs whose second warpgroup has none), with statistics."""
    import b3d.conv as C
    H = 3 * _sms() if items == "odd_per_cta" else 4             # one 128-pixel item per output row
    x, w = _operands(1, 64, H, 128 + k - 1, 64, k, H + k)
    st = torch.zeros(128, device=DEV, dtype=torch.float64)
    y = _log(lambda: C._fprop(x, C.taps_layout(w), None, k, k, k // 2, 1, stats=st))
    ref = _ref_fwd(x, w, None, k // 2, 1)
    _close(_sub(y), ref, items)
    _check_stats(st, y, 64)


def test_every_64_wide_variant_was_exercised():
    """The 64-output-channel instances cfg3 dispatches all ran in the cases above."""
    need = {"conv_wgmma<64,8>", "conv_wgmma_rowwin<64,3,4>", "conv_wgmma_rowwin<64,5,3>", "conv_wgmma_rowwin<64,2,5>"}
    missing = need - SEEN
    assert not missing, f"64-wide variants no case reached: {sorted(missing)}; seen: {sorted(SEEN)}"
