"""Input gradients with the fused LeakyReLU adjoint (b3d_conv_opts.mask, the discriminators' backward chain): the epilogues of
the three tile widths of conv_wgmma_kernel (64: weights as the M operand; 128; 256) load the mask in batches ahead of its
use and prefetch the item's mask tile into L2 before the main loop.

Against an fp64 convolution x LeakyReLU'(mask) of two images of the batch, at the tolerances of test_conv64_gpu.py, with
mask values of exactly 0, -0.0 (both: slope 1) and NaN (the slope, as !(m >= 0)) sprinkled in: each tile width at batch 32
and 64, the merged stride-2 parity classes with a 129-wide class (main launch + 1-column strip), a pitched dY, bias sums
present and absent, tiles with pixels outside the image, and channel counts below the tile width."""
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 4e-3
DEV = "cuda:0"
SLOPE = 0.2
SEEN = set()
REF_IMGS = (0, -1)          # images of the batch compared against the fp64 reference


def _log(fn):
    import b3d.conv as C
    C.VARIANT_LOG = []
    try:
        out = fn()
        torch.cuda.synchronize()
        ran = set(C.VARIANT_LOG)
    finally:
        C.VARIANT_LOG = None
    SEEN.update(ran)
    return out, ran


def _mask(shape, seed):
    """Random activations with exact zeros, negative zeros and NaNs among them."""
    m = torch.randn(shape, generator=torch.Generator().manual_seed(seed))
    flat = m.view(-1)
    flat[0::5] = 0.0
    flat[1::7] = -0.0
    flat[2::11] = float("nan")
    return m.to(DEV)


def _run(N, Cin, H, W, Cout, k, pad_y, stride, sums, pitched, seed):
    """gx of the masked input gradient, its fp64 reference on REF_IMGS, the sums tensor, the mask, the instances that ran."""
    import b3d.conv as C
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).to(DEV)
    wf = w.permute(2, 3, 0, 1).reshape(k * k, Cout, Cin)
    Hout, Wout = (H + 2 * pad_y - k) // stride + 1, (W - k) // stride + 1
    if pitched:
        gbuf = torch.randn(N, Hout, Wout + 2, Cout, generator=g).to(DEV)
        gy = gbuf[:, :, 1:Wout + 1]
    else:
        gy = torch.randn(N, Hout, Wout, Cout, generator=g).to(DEV)
    mask = _mask((N, H, W, Cin), seed + 1)
    st = torch.zeros(2 * Cin, device=DEV, dtype=torch.float64) if sums else None
    gx, ran = _log(lambda: C._dgrad(gy, C._d_layout(wf), (H, W), k, k, pad_y, stride, g_pitch=(Wout + 2) if pitched else 0,
                                    mask=mask, slope=SLOPE, sums=st))
    idx = list(REF_IMGS)
    r = torch.nn.grad.conv2d_input((len(idx), Cin, H, W), w.double(), gy[idx].permute(0, 3, 1, 2).double(), stride=stride,
                                   padding=(pad_y, 0)).permute(0, 2, 3, 1)
    r = r * torch.where(mask[idx] >= 0, 1.0, SLOPE).double()
    return gx, r, st, ran


def _check(gx, r, st, what):
    got = gx[list(REF_IMGS)]
    assert got.shape == r.shape, (what, tuple(got.shape), tuple(r.shape))
    assert bool(torch.isfinite(gx).all()), what
    err, ref = float((got.double() - r).abs().max()), float(r.abs().max())
    assert err <= TOL * ref, (what, err, ref)
    if st is not None:      # sums only: the bias gradient of the fused adjoint
        C = gx.shape[-1]
        gd = gx.double().reshape(-1, C)
        assert float((st[:C] - gd.sum(0)).abs().max()) <= 2e-6 * float(gd.abs().sum(0).max()), what
        assert float(st[C:].abs().max()) == 0.0, what


# name, Cin (channels of gx and of the mask), H, W (x-padded input), Cout, k, pad_y, stride, instances that must run
GEOM = [
    # 64-wide tiles; four merged parity classes of width 129: row window + 1-column strip
    ("d1.conv2", 64, 32, 258, 128, 4, 1, 2, {"conv_wgmma_rowwin<64,2,5>", "conv_wgmma<64,8>"}),
    # 128-wide tiles, the same structure
    ("d1.conv3.wide", 128, 16, 258, 256, 4, 1, 2, {"conv_wgmma_rowwin<128,2,4>", "conv_wgmma<128,6>"}),
    # 128-wide tiles at the layer's own width (classes of 65 columns: 64 + strip, several rows per tile)
    ("d1.conv3", 128, 32, 130, 256, 4, 1, 2, {"conv_wgmma<128,6>"}),
    # 256-wide tiles (classes of 33 columns: 32 + strip)
    ("d1.conv4", 256, 32, 66, 512, 4, 1, 2, {"conv_wgmma<256,4>"}),
    # stride 1, 3x3 row windows of both widths (width 130: main + 2-column strip)
    ("s1.3x3.64", 64, 16, 130, 64, 3, 1, 1, {"conv_wgmma_rowwin<64,3,4>", "conv_wgmma<64,8>"}),
    ("s1.3x3.128", 128, 16, 130, 128, 3, 1, 1, {"conv_wgmma_rowwin<128,3,3>", "conv_wgmma<128,6>"}),
]


@pytest.mark.parametrize("N", [32, 64])
@pytest.mark.parametrize("name,Cin,H,W,Cout,k,pad_y,stride,need", GEOM, ids=[c[0] for c in GEOM])
def test_masked_input_gradient(name, Cin, H, W, Cout, k, pad_y, stride, need, N):
    """Batch 32 without bias sums (generator step), batch 64 with them and a pitched dY (discriminator step)."""
    d_step = N == 64
    gx, r, st, ran = _run(N, Cin, H, W, Cout, k, pad_y, stride, sums=d_step, pitched=d_step, seed=sum(map(ord, name)) + N)
    assert need <= ran, (name, sorted(ran))
    _check(gx, r, st, name)


@pytest.mark.parametrize("Cin,need", [(32, "conv_wgmma<64,8>"), (96, "conv_wgmma<128,6>")], ids=["32_of_64", "96_of_128"])
@pytest.mark.parametrize("sums", [False, True])
def test_tile_and_channel_tails(Cin, need, sums):
    """5 x 40 images, 3x3 stride 1: tiles of 32 x 4 pixels, so the second tile column has 8 of 32 columns and the second tile
    row 1 of 4 rows inside the image; fewer channels than the tile is wide."""
    gx, r, st, ran = _run(3, Cin, 5, 40, 64, 3, 1, 1, sums=sums, pitched=False, seed=Cin + sums)
    assert ran == {need}, sorted(ran)
    _check(gx, r, st, f"tails {Cin}")


def test_mask_rule_is_exact():
    """0 and -0.0 keep the gradient, NaN and negatives take the slope: gx(mask) == gx(+1 everywhere) * factor, bit for bit
    (both runs have the same accumulators; the factor is 1 or the slope, applied by one multiply)."""
    import b3d.conv as C
    N, Cin, H, W, Cout = 2, 64, 8, 130, 64
    g = torch.Generator().manual_seed(5)
    wd = C._d_layout((torch.randn(9, Cout, Cin, generator=g) * 0.05).to(DEV))
    gy = torch.randn(N, H, W - 2, Cout, generator=g).to(DEV)
    mask = _mask((N, H, W, Cin), 6)
    run = lambda m: C._dgrad(gy, wd, (H, W), 3, 3, 1, 1, mask=m, slope=SLOPE)
    plain, masked = run(torch.ones_like(mask)), run(mask)
    factor = torch.where(mask >= 0, 1.0, SLOPE).float()
    assert int((factor != 1).sum()) > 0 and int((mask == 0).sum()) > 0 and int(torch.isnan(mask).sum()) > 0
    assert torch.equal(masked, plain * factor)


def test_every_masked_variant_was_exercised():
    need = set().union(*(c[-1] for c in GEOM))
    missing = need - SEEN
    assert not missing, f"instances no masked case reached: {sorted(missing)}; seen: {sorted(SEEN)}"
