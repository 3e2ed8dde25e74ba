"""wgmma implicit-GEMM conv (tf32) against torch's fp32 conv2d (TF32 disabled) on the same inputs.
Tolerance: tf32 keeps 10 mantissa bits (the tensor core truncates fp32 operands), so each product carries
<= 2^-9 relative error; we require max |err| <= 4e-3 * max|ref| (cuDNN's TF32 path, the reference's default
on Ampere+, is in the same class)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 4e-3


def ref_conv(x_nchw, w, b, pad_y, stride):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.nn.functional.conv2d(x_nchw, w, b, stride=stride, padding=(pad_y, 0))


CASES = [  # N, Cin, H, W(x-padded), Cout, k, pad_y, stride, bias, leaky
    (2, 64, 8, 16, 64, 1, 0, 1, False, 1.0),        # pure GEMM, one tile per image
    (2, 128, 16, 18, 128, 3, 1, 1, False, 1.0),     # ResBlockUp conv (gan.py:294)
    (3, 512, 8, 6, 512, 3, 1, 1, False, 1.0),       # blk1: 8x4 images, 4 images per tile, 2 N tiles x 4 Cout tiles
    (2, 64, 32, 36, 3, 5, 2, 1, True, 1.0),         # conv_final 5x5 -> 3 channels (gan.py:359)
    (2, 32, 32, 34, 64, 4, 1, 2, True, 0.2),        # discriminator 4x4 / stride 2 + bias + LeakyReLU (gan.py:163)
    (1, 256, 64, 66, 128, 3, 1, 1, False, 1.0),     # multiple tiles along y
    (5, 96, 10, 20, 40, 3, 1, 1, True, 1.0),        # ragged: N, H, Cout not multiples of the tile
    (2, 64, 32, 34, 128, 3, 1, 2, False, 1.0),      # reconstruction encoder: 3x3 / stride 2 (reconstruction.py:54-60)
    (2, 32, 32, 36, 64, 5, 2, 2, False, 1.0),       # ... and its 5x5 / stride 2 stem (:52)
]


@pytest.mark.parametrize("N,Cin,H,W,Cout,k,pad_y,stride,bias,leaky", CASES)
def test_fprop(N, Cin, H, W, Cout, k, pad_y, stride, bias, leaky):
    from b3d.conv import conv2d_nhwc
    g = torch.Generator().manual_seed(Cin + Cout + k)
    x = torch.randn(N, Cin, H, W, generator=g).cuda()
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda()
    b = torch.randn(Cout, generator=g).cuda() if bias else None
    ref = torch.nn.functional.leaky_relu(ref_conv(x, w, b, pad_y, stride), leaky) if leaky != 1.0 else ref_conv(x, w, b, pad_y, stride)
    out = conv2d_nhwc(x.permute(0, 2, 3, 1).contiguous(), w, b, pad_y=pad_y, stride=stride, leaky=leaky)
    torch.cuda.synchronize()
    out = out.permute(0, 3, 1, 2)
    assert out.shape == ref.shape
    err = float((out - ref).abs().max())
    assert err <= TOL * float(ref.abs().max()), (err, float(ref.abs().max()))


@pytest.mark.parametrize("N,Cin,H,W,Cout,k,pad_y,stride", [
    (2, 64, 16, 18, 128, 3, 1, 1), (2, 32, 32, 36, 64, 5, 2, 1), (2, 64, 16, 18, 64, 4, 1, 2), (3, 128, 8, 6, 256, 3, 1, 1),
    (2, 96, 9, 12, 64, 1, 0, 1), (2, 64, 32, 34, 128, 3, 1, 2), (2, 128, 16, 18, 256, 3, 1, 2), (2, 32, 16, 20, 64, 5, 2, 2),
])
def test_dgrad(N, Cin, H, W, Cout, k, pad_y, stride):
    from b3d.conv import conv2d_dgrad_nhwc
    g = torch.Generator().manual_seed(Cin * 3 + Cout + k)
    x = torch.randn(N, Cin, H, W, generator=g).cuda().requires_grad_(True)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda()
    y = ref_conv(x, w, None, pad_y, stride)
    gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(1)).cuda()
    ref, = torch.autograd.grad(y, x, gy)
    out = conv2d_dgrad_nhwc(gy.permute(0, 2, 3, 1).contiguous(), w, (H, W), pad_y=pad_y, stride=stride)
    torch.cuda.synchronize()
    out = out.permute(0, 3, 1, 2)
    err = float((out - ref).abs().max())
    assert err <= TOL * float(ref.abs().max()), (err, float(ref.abs().max()))


@pytest.mark.parametrize("N,Cin,H,W,Cout,k,pad_y,stride", [
    (2, 64, 16, 18, 128, 3, 1, 1), (4, 128, 64, 66, 64, 3, 1, 1), (2, 32, 32, 36, 4, 5, 2, 1), (2, 64, 16, 18, 64, 4, 1, 2),
    (3, 512, 8, 6, 512, 3, 1, 1), (2, 96, 9, 12, 40, 1, 0, 1), (8, 32, 64, 66, 64, 4, 1, 2),
    (2, 64, 32, 34, 128, 3, 1, 2), (2, 32, 32, 36, 64, 5, 2, 2), (4, 256, 4, 4, 512, 3, 1, 1),
])
def test_wgrad(N, Cin, H, W, Cout, k, pad_y, stride):
    from b3d.conv import conv2d_wgrad_nhwc
    g = torch.Generator().manual_seed(Cin * 5 + Cout + k)
    x = torch.randn(N, Cin, H, W, generator=g).cuda()
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda().requires_grad_(True)
    y = ref_conv(x, w, None, pad_y, stride)
    gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(2)).cuda()
    ref, = torch.autograd.grad(y, w, gy)
    out = conv2d_wgrad_nhwc(gy.permute(0, 2, 3, 1).contiguous(), x.permute(0, 2, 3, 1).contiguous(), k, k, pad_y=pad_y,
                            stride=stride)
    torch.cuda.synchronize()
    err = float((out - ref).abs().max())
    assert err <= TOL * float(ref.abs().max()), (err, float(ref.abs().max()))


@pytest.mark.parametrize("N,Cin,H,W,Cout,k,pad_y,stride,bias", [
    (2, 8, 32, 36, 64, 5, 2, 1, True),       # discriminator stem, 8 channels: kw folded into K
    (2, 11, 32, 36, 64, 5, 2, 1, True),      # mesh discriminator stem, 11 channels
    (2, 8, 32, 34, 64, 4, 1, 2, True),       # 512^2 stem: 4x4 / stride 2 (channels zero-padded to 32)
    (2, 64, 16, 20, 3, 5, 2, 1, True),       # 3-channel head (CUDA-core thin kernels for fprop / wgrad)
    (3, 512, 9, 13, 1, 5, 2, 1, True),       # discriminator head 512 -> 1
    (2, 256, 8, 12, 1, 5, 2, 1, False),      # mesh discriminator head 256 -> 1
    (2, 128, 6, 9, 2, 5, 2, 1, True),
    (2, 256, 16, 18, 128, 3, 1, 1, False),
    (2, 4, 64, 68, 64, 5, 2, 2, False),      # reconstruction stem: 4 input channels, 5x5 / stride 2
    (4, 256, 4, 4, 256, 3, 1, 1, False),     # decoder base resolution: 4x2 maps (x-padded to 4)
])
def test_conv2d_autograd_matches_torch(N, Cin, H, W, Cout, k, pad_y, stride, bias):
    """b3d.conv.conv2d (the function models/gan.py calls) forward + all three gradients vs torch fp32."""
    from b3d.conv import conv2d
    g = torch.Generator().manual_seed(Cin * 7 + Cout)
    x0 = torch.randn(N, Cin, H, W, generator=g).cuda()
    w0 = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda()
    b0 = torch.randn(Cout, generator=g).cuda() if bias else None
    outs = []
    for impl in ("torch", "b3d"):
        x, w = x0.clone().requires_grad_(True), w0.clone().requires_grad_(True)
        b = b0.clone().requires_grad_(True) if bias else None
        y = ref_conv(x, w, b, pad_y, stride) if impl == "torch" else conv2d(x.contiguous(memory_format=torch.channels_last), w, b, pad_y, stride)
        gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(3)).cuda()
        grads = torch.autograd.grad(y, [x, w] + ([b] if bias else []), gy)
        outs.append([y.detach()] + list(grads))
    for a, r in zip(outs[1], outs[0]):
        assert a.shape == r.shape
        assert float((a - r).abs().max()) <= TOL * float(r.abs().max()), (a.shape, float((a - r).abs().max()), float(r.abs().max()))


@pytest.mark.parametrize("N,Cin,H,W,Cout,k,pad_y,stride", [
    (2, 64, 16, 18, 128, 3, 1, 1),      # 3x3 stride 1
    (2, 64, 16, 18, 128, 4, 1, 2),      # 4x4 stride 2 on an even-sized input: one launch over the four parity classes
    (2, 256, 12, 16, 1, 5, 2, 1),       # 1-channel 5x5 head (CUDA-core thin kernels for fprop / wgrad)
])
def test_module_and_bank_entries_agree(N, Cin, H, W, Cout, k, pad_y, stride):
    """One plain TCConv2d through conv2d (per-call layouts of the module weight) and through conv2d_banked (WeightBank
    layouts without tf32 rounding): the same kernels on the same fp32 weights, so forward outputs, input and bias gradients
    are bitwise equal; weight gradients differ only by the order of the split-K fp32 atomics."""
    from b3d.bank import WeightBank
    from b3d.conv import conv2d, conv2d_banked
    from models.gan import TCConv2d
    torch.manual_seed(Cin + Cout + k)
    conv = TCConv2d(Cin, Cout, k, padding=(pad_y, 0), stride=stride).cuda()
    x0 = torch.randn(N, Cin, H, W, device="cuda").contiguous(memory_format=torch.channels_last)
    gy = None
    res = []
    for banked in (False, True):
        conv.zero_grad()
        x = x0.detach().clone().requires_grad_(True)
        if banked:
            y = conv2d_banked(x, WeightBank({"c": conv}, round_tf32=False).forward(True)["c"], pad_y=pad_y, stride=stride)
        else:
            y = conv2d(x, conv.weight, conv.bias, pad_y, stride)
        if gy is None:
            gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(3)).cuda()
        y.backward(gy)
        res.append((y.detach(), x.grad, conv.bias.grad.clone(), conv.weight.grad.clone()))
    torch.cuda.synchronize()
    (ym, gxm, gbm, gwm), (yb, gxb, gbb, gwb) = res
    assert torch.equal(ym, yb) and torch.equal(gxm, gxb) and torch.equal(gbm, gbb)
    assert float((gwm - gwb).abs().max()) <= 1e-5 * float(gwm.abs().max())


@pytest.mark.parametrize("mode", ["replicate", "circular"])
@pytest.mark.parametrize("N,C,H,W,a", [(2, 8, 5, 7, 2), (3, 64, 16, 4, 1), (1, 12, 3, 9, 2)])
def test_pad_x_matches_torch(mode, N, C, H, W, a):
    from b3d.ew import CIRCULAR, REPLICATE, pad_x
    g = torch.Generator().manual_seed(N * C + W)
    x0 = torch.randn(N, C, H, W, generator=g).cuda()
    outs = []
    for impl in (0, 1):
        x = x0.clone().contiguous(memory_format=torch.channels_last).requires_grad_(True)
        if impl == 0:
            y = torch.nn.functional.pad(x, (a, a, 0, 0), mode=mode)
        else:
            y = pad_x(x, a, REPLICATE if mode == "replicate" else CIRCULAR)
        gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(4)).cuda()
        gx, = torch.autograd.grad(y, x, gy)
        outs.append((y.detach(), gx))
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.allclose(outs[0][1], outs[1][1], atol=1e-6)


def test_fused_leaky_epilogue_autograd():
    from b3d.conv import conv2d
    g = torch.Generator().manual_seed(9)
    x0 = torch.randn(2, 64, 16, 18, generator=g).cuda()
    w0 = (torch.randn(128, 64, 4, 4, generator=g) / 32).cuda()
    b0 = torch.randn(128, generator=g).cuda()
    res = []
    for impl in (0, 1):
        x, w, b = x0.clone().requires_grad_(True), w0.clone().requires_grad_(True), b0.clone().requires_grad_(True)
        if impl == 0:
            y = torch.nn.functional.leaky_relu(ref_conv(x, w, b, 1, 2), 0.2)
        else:
            y = conv2d(x.contiguous(memory_format=torch.channels_last), w, b, 1, 2, leaky=0.2)
        gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(5)).cuda()
        res.append([y.detach()] + list(torch.autograd.grad(y, [x, w, b], gy)))
    for a, r in zip(res[1], res[0]):
        assert float((a - r).abs().max()) <= 2 * TOL * float(r.abs().max())


@pytest.mark.parametrize("mode", ["replicate", "circular"])
@pytest.mark.parametrize("N,Cin,H,W,Cout,k,pad_y,stride,pad_out,bias", [
    (2, 64, 16, 18, 128, 4, 1, 2, 1, True),      # discriminator conv2 -> next 4x4 layer's padding
    (3, 8, 24, 28, 64, 5, 2, 1, 1, True),        # folded stem -> padded by 1
    (2, 128, 8, 10, 256, 4, 1, 2, 2, False),     # conv4 -> the 5x5 head's padding of 2
    (1, 32, 140, 134, 64, 3, 1, 1, 2, True),     # wide rows: main + strip launches into the padded buffer
])
def test_conv_leaky_pad_fused_autograd(mode, N, Cin, H, W, Cout, k, pad_y, stride, pad_out, bias):
    """conv -> bias -> LeakyReLU -> x padding in one op (epilogue writes the padded buffer, one fused backward pass)
    against the same chain in plain torch fp32 (models/gan.py discriminators :163-177, :294-302)."""
    from b3d.conv import conv2d
    from b3d.ew import CIRCULAR, REPLICATE
    g = torch.Generator().manual_seed(Cin * 3 + Cout + pad_out)
    x0 = torch.randn(N, Cin, H, W, generator=g).cuda()
    w0 = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda()
    b0 = torch.randn(Cout, generator=g).cuda() if bias else None
    outs, mask = [], None
    for impl in ("b3d", "torch"):
        x, w = x0.clone().requires_grad_(True), w0.clone().requires_grad_(True)
        b = b0.clone().requires_grad_(True) if bias else None
        if impl == "torch":
            # pre-activations within tf32 rounding of zero may change sign between the two implementations; the
            # reference chain takes the activation mask of the kernel's output so that gradients are comparable
            z = ref_conv(x, w, b, pad_y, stride)
            y = torch.where(mask, z, 0.2 * z)
            y = torch.nn.functional.pad(y, (pad_out, pad_out, 0, 0), mode=mode)
        else:
            y = conv2d(x.contiguous(memory_format=torch.channels_last), w, b, pad_y, stride, leaky=0.2, pad_out=pad_out,
                       pad_mode=REPLICATE if mode == "replicate" else CIRCULAR)
            mask = y.detach()[..., pad_out:y.shape[3] - pad_out] >= 0
        gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(5)).cuda()
        grads = torch.autograd.grad(y, [x, w] + ([b] if bias else []), gy)
        outs.append([y.detach()] + list(grads))
    for a, r in zip(outs[0], outs[1]):
        assert a.shape == r.shape
        assert float((a - r).abs().max()) <= TOL * float(r.abs().max()), (a.shape, float((a - r).abs().max()), float(r.abs().max()))


@pytest.mark.parametrize("N,C,H,W,kh,pad_y", [(2, 8, 12, 9, 5, 2), (3, 11, 7, 5, 5, 2), (1, 4, 6, 6, 3, 0)])
def test_fold_rows_matches_torch(N, C, H, W, kh, pad_y):
    """b3d_fold_rows_fwd/_bwd (thin-stem fold of the vertical taps into channels) against slicing + cat."""
    from b3d.ew import fold_rows
    g = torch.Generator().manual_seed(N + C)
    x0 = torch.randn(N, H, W, C, generator=g).cuda()
    Cp = -(-kh * C // 32) * 32
    Hout = H + 2 * pad_y - kh + 1
    outs = []
    for impl in (0, 1):
        x = x0.clone().requires_grad_(True)
        if impl == 0:
            xp = torch.nn.functional.pad(x, (0, 0, 0, 0, pad_y, pad_y))
            y = torch.cat([xp[:, r:r + Hout] for r in range(kh)] + [x.new_zeros(N, Hout, W, Cp - kh * C)], dim=3)
        else:
            y = fold_rows(x, kh, pad_y, Cp)
        gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(6)).cuda()
        gx, = torch.autograd.grad(y, x, gy)
        outs.append((y.detach(), gx))
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.allclose(outs[0][1], outs[1][1], atol=1e-5)


@pytest.mark.parametrize("N,Cin,H,W,Cout,k,pad_y", [(2, 128, 16, 34, 64, 1, 0), (2, 64, 8, 20, 64, 3, 1)])
def test_conv2d_x_crop_autograd(N, Cin, H, W, Cout, k, pad_y):
    """conv2d(x, w, x_crop=1) == conv2d(x[..., 1:-1], w) with gradients w.r.t. the full padded input (the ResBlockUp
    1x1 shortcut reads the interior of the replicate-padded block input, models/gan.py:233-246)."""
    from b3d.conv import conv2d
    g = torch.Generator().manual_seed(Cin + Cout + k)
    x0 = torch.randn(N, Cin, H, W, generator=g).cuda()
    w0 = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda()
    outs = []
    for impl in ("torch", "b3d"):
        x, w = x0.clone().requires_grad_(True), w0.clone().requires_grad_(True)
        if impl == "torch":
            y = ref_conv(x[..., 1:-1], w, None, pad_y, 1)
        else:
            y = conv2d(x.contiguous(memory_format=torch.channels_last), w, None, pad_y, 1, x_crop=1)
        gy = torch.randn(y.shape, generator=torch.Generator().manual_seed(7)).cuda()
        outs.append([y.detach()] + list(torch.autograd.grad(y, [x, w], gy)))
    for a, r in zip(outs[1], outs[0]):
        assert a.shape == r.shape
        assert float((a - r).abs().max()) <= TOL * float(r.abs().max()), (a.shape, float((a - r).abs().max()), float(r.abs().max()))
