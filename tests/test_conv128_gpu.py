"""The 128- and 256-output-channel tiles of the wgmma convolution (conv_wgmma<128,6>, conv_wgmma_rowwin<128,KW,S> and
conv_wgmma<256,4>): weights as the wgmma M operand in 64-channel blocks, 128-pixel tiles as the N operand; 128-wide items
alternate between the two consumer warpgroups, a 256-wide item is shared, one 128-channel half per warpgroup.

Every 128- and 256-wide geometry cfg3 dispatches, at batch 32 and 64, forward and input gradient, against an fp64
convolution of two images of the batch; epilogue statistics against the sums of the stored output (the bounds of
test_bench_shapes_gpu.py::test_epilogue_statistics).  Also the epilogue's edges: the fused LeakyReLU adjoint (mask) with
sums-only statistics, a pitched dY, the four merged parity classes, strip launches (widths 130 and 129), pad_out, x_crop,
output-channel counts that are not a multiple of 128 (the Inception widths: the weight box overhangs, and at 192 a whole
64-channel block of the last tile is empty), CTAs with an odd number of items and grids with fewer items than SMs."""
import pytest
import torch

from test_conv64_gpu import _check_stats, _close, _mask_like, _operands, _ref_dgrad, _ref_fwd, _sub

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEEN = set()


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


# name, Cin, H, W (x-padded input), Cout, k, pad_y, stride, x_crop — the 128- and 256-wide forward launches of cfg3
FWD = [("G.blk1.conv", 512, 8, 6, 512, 3, 1, 1, 0),
       ("G.blk2.conv1", 512, 16, 10, 256, 3, 1, 1, 0),
       ("G.blk2.short", 512, 16, 10, 256, 1, 0, 1, 1),
       ("G.blk3a.conv", 256, 32, 18, 256, 3, 1, 1, 0),
       ("G.blk4.conv1", 256, 64, 34, 128, 3, 1, 1, 0),
       ("G.blk4.short", 256, 64, 34, 128, 1, 0, 1, 1),
       ("G.blk5.conv", 128, 128, 66, 128, 3, 1, 1, 0),               # rowwin<128,3,3> + 2-column strip
       ("D1.conv2", 64, 256, 258, 128, 4, 1, 2, 0),
       ("D1.conv3", 128, 128, 130, 256, 4, 1, 2, 0),
       ("D1.conv4", 256, 64, 66, 512, 4, 1, 2, 0),
       ("D2.conv3", 128, 16, 18, 256, 4, 1, 2, 0)]


# statistics: the stride-1 (generator) layers only, as b3d.conv allows
FWD_CASES = [c + (stats,) for c in FWD for stats in ((False, True) if c[7] == 1 else (False,))]


@pytest.mark.parametrize("N", [32, 64])
@pytest.mark.parametrize("name,Cin,H,W,Cout,k,pad_y,stride,x_crop,stats", FWD_CASES,
                         ids=[c[0] + ("-stats" if c[-1] else "") for c in FWD_CASES])
def test_forward(name, Cin, H, W, Cout, k, pad_y, stride, x_crop, stats, N):
    import b3d.conv as C
    x, w = _operands(N, Cin, H, W, Cout, k, sum(map(ord, name)) + N)
    st = torch.zeros(2 * Cout, device=DEV, dtype=torch.float64) if stats else None
    y = _log(lambda: C._fprop(x, C.taps_layout(w), None, k, k, pad_y, stride, x_crop=x_crop, stats=st))
    _close(_sub(y), _ref_fwd(x, w, None, pad_y, stride, x_crop), name)
    if stats:
        _check_stats(st, y, Cout)


@pytest.mark.parametrize("Cout", [128, 256])
def test_forward_bias_leaky_pad_out(Cout):
    """bias + LeakyReLU in the epilogue, written into the interior of an x-padded buffer (main + 2-column strip launch)."""
    import b3d.conv as C
    N, W, pad_out = 64, 130, 1
    x, w = _operands(N, 64, 64, W, Cout, 3, W + Cout)
    b = torch.randn(Cout, generator=torch.Generator().manual_seed(1)).to(DEV)
    y = _log(lambda: C._fprop(x, C.taps_layout(w), b, 3, 3, 1, 1, leaky=0.2, pad_out=pad_out))
    r = _ref_fwd(x, w, b, 1, 1)
    _close(_sub(y)[:, :, pad_out:y.shape[2] - pad_out], torch.where(r >= 0, r, 0.2 * r), "bias/leaky/pad_out")


@pytest.mark.parametrize("Cout", [96, 192, 320, 384, 448])
def test_forward_partial_channel_tiles(Cout):
    """Output-channel counts of the Inception network: the last tile's weight box overhangs Cout (TMA's zero fill), and
    with 192 its second 64-channel block holds no channel at all; statistics and bias only over the real channels."""
    import b3d.conv as C
    x, w = _operands(4, 64, 35, 35, Cout, 3, Cout)
    b = torch.randn(Cout, generator=torch.Generator().manual_seed(2)).to(DEV)
    y = _log(lambda: C._fprop(x, C.taps_layout(w), b, 3, 3, 1, 1))
    _close(_sub(y), _ref_fwd(x, w, b, 1, 1), f"Cout={Cout}")
    st = torch.zeros(2 * Cout, device=DEV, dtype=torch.float64)          # statistics: of the output before any bias
    y = _log(lambda: C._fprop(x, C.taps_layout(w), None, 3, 3, 1, 1, stats=st))
    _check_stats(st, y, Cout)


# name, Cin (input-gradient channels), H, W, Cout (dY channels), k, pad_y, stride, x_crop, masked, pitched
DGRAD = [("D1.conv3", 128, 128, 130, 256, 4, 1, 2, 0, True, False),      # four parity classes of width 65: 64 + 1-column strip
         ("D1.conv4", 256, 64, 66, 512, 4, 1, 2, 0, True, True),        # 256-wide at batch 64, parity classes of width 33
         ("D1.conv3.wide", 128, 64, 258, 128, 4, 1, 2, 0, True, False),  # parity classes of width 129: main + 1-column strip
         ("G.blk3a.conv", 256, 32, 18, 256, 3, 1, 1, 0, False, False),
         ("G.blk4.conv1", 256, 64, 34, 128, 3, 1, 1, 0, False, True),
         ("G.blk4.short", 256, 64, 34, 128, 1, 0, 1, 1, False, False),    # x_crop
         ("G.blk5.conv", 128, 128, 66, 128, 3, 1, 1, 0, False, False),
         ("G.blk6.conv1", 128, 256, 130, 64, 3, 1, 1, 0, True, True),     # rowwin<128,3,3>: width 130 = main + strip launch
         ("k5.masked", 128, 32, 132, 64, 5, 2, 1, 0, True, False)]       # rowwin<128,5,2>: 4 mask stages through a 2-stage ring


@pytest.mark.parametrize("N", [32, 64])
@pytest.mark.parametrize("name,Cin,H,W,Cout,k,pad_y,stride,x_crop,masked,pitched", DGRAD, ids=[c[0] for c in DGRAD])
def test_input_gradient(name, Cin, H, W, Cout, k, pad_y, stride, x_crop, masked, pitched, N):
    """Input gradient with 128 or 256 output channels (= the layer's input channels): the mask (LeakyReLU adjoint of the
    input's activation, slope 0.2) and the sums-only statistics of the fused adjoint, dY read in place from a padded buffer."""
    import b3d.conv as C
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


@pytest.mark.parametrize("Cout", [128, 256])
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("items", ["odd_per_cta", "fewer_than_sms"])
def test_work_distribution(items, k, Cout):
    """128-wide items alternate between the two consumer warpgroups of a CTA, 256-wide ones are shared: three items per
    CTA, and a grid of fewer items than SMs (128-wide: CTAs whose second warpgroup has none; 256-wide tiles are not chosen
    for such a grid, so it runs 128-wide), with statistics."""
    import b3d.conv as C
    H = 3 * _sms() if items == "odd_per_cta" else 4             # one 128-pixel item per output row and channel tile
    x, w = _operands(1, 64, H, 128 + k - 1, Cout, k, H + k + Cout)
    st = torch.zeros(2 * Cout, device=DEV, dtype=torch.float64)
    y = _log(lambda: C._fprop(x, C.taps_layout(w), None, k, k, k // 2, 1, stats=st))
    ref = _ref_fwd(x, w, None, k // 2, 1)
    _close(_sub(y), ref, items)
    _check_stats(st, y, Cout)


def test_every_128_and_256_wide_variant_was_exercised():
    """The 128- and 256-output-channel instances cfg3 dispatches, and the 5-tap row window, all ran in the cases above."""
    need = {"conv_wgmma<128,6>", "conv_wgmma<256,4>", "conv_wgmma_rowwin<128,3,3>", "conv_wgmma_rowwin<128,2,4>",
            "conv_wgmma_rowwin<128,5,2>"}
    missing = need - SEEN
    assert not missing, f"128- and 256-wide variants no case reached: {sorted(missing)}; seen: {sorted(SEEN)}"
