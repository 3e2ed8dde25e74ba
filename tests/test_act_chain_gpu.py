"""The discriminators' chained backward pass (b3d.conv.ActLink): LeakyReLU', the wrap-around padding's adjoint and the bias
sum of layer L applied in the input-gradient epilogue of layer L+1 (`b3d_conv_opts.mask`, b3d_wrap_x_bwd_inplace), the
padded gradient read in place through row-pitch tensor maps (`x_row_pitch`, `dy_row_pitch`).

Checked three ways: (1) the ABI extras one by one against torch on the same operands (the mask / pitch / fold-back are exact
re-arrangements of the same fp32 values, so the tolerance is the tf32 conv's own: 4e-3 of the largest magnitude vs an fp64
convolution, and 1e-6 where both sides run the same kernel); (2) a whole MultiScaleDiscriminator backward with the chain
on against the same network with the chain off (stand-alone b3d_pad_leaky_bias_bwd passes): every parameter gradient and
the input gradient to 5e-4 of the largest magnitude (the pad fold-back adds a*m + b*m instead of (a + b)*m and the bias sums are
fp64 instead of fp32 atomics: last-bit differences of the gradient that the next layer's tf32 operand rounding amplifies to
~2^-11 relative on single elements); (3) tests/test_gan_gpu.py pins the chained path to the reference's golden gradients at B = 2 / 32 / 512^2."""
import ctypes
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import gan_common as GC          # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _close(a, b, tol, what=""):
    scale = max(float(b.abs().max()), 1e-12)
    err = float((a.double() - b.double()).abs().max())
    assert err <= tol * scale, (what, err, tol * scale)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("amount", [1, 2])
def test_wrap_x_bwd_inplace_is_the_adjoint_of_the_padding(mode, amount):
    from b3d import check, lib, ptr, stream_ptr
    from b3d.ew import pad_x
    torch.manual_seed(0)
    rows, W, C = 6, 10, 8
    x = torch.randn(2, C, 3, W, device=DEV, requires_grad=True)
    g = torch.randn(2, C, 3, W + 2 * amount, device=DEV)
    want, = torch.autograd.grad(pad_x(x, amount, mode), x, g)
    buf = g.permute(0, 2, 3, 1).contiguous()                    # [rows, W + 2a, C]
    check(lib.b3d_wrap_x_bwd_inplace(ptr(buf), rows, W, C, amount, mode, stream_ptr(buf)))
    got = buf[:, :, amount:amount + W].permute(0, 3, 1, 2)
    _close(got, want, 1e-6)
    assert torch.equal(buf[:, :, :amount], g.permute(0, 2, 3, 1)[:, :, :amount])      # pad columns untouched


def _conv_args(x, wt, out, Hout, Wout, dy, dx, stats, opts):
    from b3d import ptr, stream_ptr
    from b3d.conv import _ints
    N, H, W, Cin = x.shape
    Cout = wt.shape[1]
    return (ptr(wt), None, ptr(out), N, H, W, Cin, Hout, Wout, Cout, len(dy), _ints(dy), _ints(dx), 1, 1, out.shape[1], out.shape[2],
            Cout, 1, 1, 0, 0, 1.0, None, 0, ptr(stats), 0, 0, ctypes.cast(ctypes.pointer(opts), ctypes.c_void_p) if opts else None,
            stream_ptr(x))


@pytest.mark.parametrize("N,H,W,Cin,Cout", [(2, 16, 130, 64, 64), (8, 80, 256, 64, 64), (1, 8, 40, 32, 128), (1, 16, 16, 256, 256)])
def test_conv_opts_mask_and_row_pitch(N, H, W, Cin, Cout):
    """3x3 stride-1 conv through b3d_conv2d_tf32 (row-window or per-tap kernel, whichever the shape dispatches) with
    (a) the activation mask + sum statistics and (b) the input read as the interior of a wider buffer."""
    from b3d import check, lib, ptr
    from b3d.conv import _ConvOpts, taps_layout
    torch.manual_seed(1)
    pad = 3
    wide = torch.randn(N, H, W + 2 * pad, Cin, device=DEV)
    xin = wide[:, :, pad:pad + W].contiguous()
    w = torch.randn(Cout, Cin, 3, 3, device=DEV) * 0.05
    wt = taps_layout(w)
    dy = [r - 1 for r in range(3) for _ in range(3)]
    dx = [s - 1 for _ in range(3) for s in range(3)]
    ref = F.conv2d(xin.permute(0, 3, 1, 2).double(), w.double(), padding=1).permute(0, 2, 3, 1)
    act = torch.randn(N, H, W, Cout, device=DEV)
    act[0, 0, 0, :4] = 0.0                                      # zeros pass (the >= 0 rule of leaky_relu's backward)
    slope = 0.2
    want = ref * torch.where(act >= 0, 1.0, slope).double()

    out = torch.empty(N, H, W, Cout, device=DEV)
    sums = torch.zeros(2 * Cout, device=DEV, dtype=torch.float64)
    opts = _ConvOpts(act.data_ptr(), slope, 1, 0, 0)
    check(lib.b3d_conv2d_tf32(ptr(xin), *_conv_args(xin, wt, out, H, W, dy, dx, sums, opts)))
    _close(out, want, 4e-3, "masked output")
    err = float((sums[:Cout] - out.double().sum(dim=(0, 1, 2))).abs().max())          # fp32 warp / CTA partials, fp64 across CTAs
    assert err <= 2e-6 * float(out.double().abs().sum(dim=(0, 1, 2)).max()), err
    assert float(sums[Cout:].abs().max()) == 0.0                # sums only

    plain = torch.empty(N, H, W, Cout, device=DEV)
    check(lib.b3d_conv2d_tf32(ptr(xin), *_conv_args(xin, wt, plain, H, W, dy, dx, None, None)))
    pitched = torch.empty(N, H, W, Cout, device=DEV)
    opts = _ConvOpts(None, 1.0, 0, W + 2 * pad, 0)
    view = wide[:, :, pad:pad + W]                              # non-contiguous: rows W + 2 pad pixels apart
    check(lib.b3d_conv2d_tf32(ctypes.c_void_p(view.data_ptr()), *_conv_args(xin, wt, pitched, H, W, dy, dx, None, opts)))
    assert torch.equal(pitched, plain)                          # same kernel, same operands (columns outside [0, W) read as zero)


@pytest.mark.parametrize("stride,kh,N,H,W,Cin,Cout", [(2, 4, 2, 32, 66, 64, 128), (1, 3, 2, 16, 34, 64, 64), (2, 4, 4, 64, 130, 64, 128)])
def test_wgrad_dy_row_pitch(stride, kh, N, H, W, Cin, Cout):
    from b3d import check, lib, ptr, stream_ptr
    torch.manual_seed(2)
    kw, pad_y = kh, 1
    Hout, Wout = (H + 2 * pad_y - kh) // stride + 1, (W - kw) // stride + 1
    x = torch.randn(N, H, W, Cin, device=DEV)
    p = 2
    wide = torch.randn(N, Hout, Wout + 2 * p, Cout, device=DEV)
    view = wide[:, :, p:p + Wout]
    dense = view.contiguous()
    a = torch.zeros(kh * kw, Cout, Cin, device=DEV)
    b = torch.zeros_like(a)
    check(lib.b3d_conv2d_wgrad_tf32(ptr(dense), ptr(x), ptr(a), N, H, W, Cin, Hout, Wout, Cout, kh, kw, pad_y, stride, 0, 1, 0, 0, stream_ptr(x)))
    check(lib.b3d_conv2d_wgrad_tf32(ctypes.c_void_p(view.data_ptr()), ptr(x), ptr(b), N, H, W, Cin, Hout, Wout, Cout, kh, kw, pad_y, stride, 0,
                                    1, 0, Wout + 2 * p, stream_ptr(x)))
    _close(b, a, 2e-5, "same kernel; split-K atomics reorder the fp32 sums")
    xd = x.permute(0, 3, 1, 2).double().requires_grad_(True)
    wd = torch.zeros(Cout, Cin, kh, kw, device=DEV, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(xd, wd, stride=stride, padding=(pad_y, 0))
    gw, = torch.autograd.grad(y, wd, dense.permute(0, 3, 1, 2).double())
    _close(b, gw.permute(2, 3, 0, 1).reshape(kh * kw, Cout, Cin), 4e-3, "vs fp64 autograd")


@pytest.mark.parametrize("res,nd,B", [(256, 2, 2), (256, 2, 8), (512, 3, 2)])
def test_chained_backward_equals_stand_alone_passes(res, nd, B):
    from models import gan
    args = GC.make_args(res, nd)
    _, D = GC.build(gan, args)
    D.cuda().train()
    z, c, alpha, tex, mesh = [t.cuda() for t in GC.inputs(args, B=B)]
    x0 = torch.cat((tex, alpha), dim=1)
    discs = [getattr(D, n) for n in ("d1", "d2", "d3") if hasattr(D, n)]
    results, passes = [], []
    from b3d import lib
    real_fn = lib.b3d_pad_leaky_bias_bwd

    def counting(*a):
        passes[-1] += 1
        return real_fn(*a)

    for chain in (False, True):
        passes.append(0)
        for d in discs:
            d.disable_act_chain = not chain
        D.zero_grad()
        for m in D.modules():                                   # the same power-iteration state for both passes
            if hasattr(m, "weight_u"):
                m._saved_uv = getattr(m, "_saved_uv", None) or (m.weight_u.clone(), m.weight_v.clone())
                m.weight_u.copy_(m._saved_uv[0]); m.weight_v.copy_(m._saved_uv[1])
        x = x0.clone().requires_grad_(True)
        mm = mesh.clone().requires_grad_(True)
        lib.b3d_pad_leaky_bias_bwd = counting
        try:
            out, _ = D(x, mm, c)
            g = torch.Generator(device="cuda").manual_seed(3)
            loss = sum((o * torch.randn(o.shape, device=o.device, generator=g)).sum() for o in out)
            loss.backward()
            torch.cuda.synchronize()
        finally:
            lib.b3d_pad_leaky_bias_bwd = real_fn
        results.append(({n: p.grad.clone() for n, p in D.named_parameters() if p.grad is not None}, x.grad.clone(), mm.grad.clone()))
    (g0, x0g, m0g), (g1, x1g, m1g) = results
    assert set(g0) == set(g1) and any(n.endswith("conv1.bias") for n in g0)
    bad = []
    for n, a, b in [(n, g1[n], g0[n]) for n in g0] + [("input gradient", x1g, x0g), ("mesh-map gradient", m1g, m0g)]:
        rel = float((a.double() - b.double()).abs().max()) / max(float(b.abs().max()), 1e-12)
        if rel > 5e-4:
            bad.append((n, round(rel, 6)))
    assert not bad, bad
    # and the chain really ran: one stand-alone pass per discriminator is left (the last padded activation also feeds the
    # projection), against one per padded layer without the chain (texture discriminators 4, mesh discriminator 3)
    assert passes[1] == len(discs) and passes[0] == sum(4 if isinstance(d, gan.TextureDiscriminator) else 3 for d in discs), passes


def test_chain_is_off_without_the_weight_bank_or_when_disabled():
    from models import gan
    args = GC.make_args(256, 2)
    _, D = GC.build(gan, args)
    assert all(lk is None for lk in D.d1._links(3, None))
    D.d1.disable_act_chain = True
    assert all(lk is None for lk in D.d1._links(3, {"x": 1}))


@pytest.mark.parametrize("res,nd,B", [(256, 2, 2), (256, 2, 16), (512, 3, 2)])
def test_merged_parity_classes_equal_per_class_launches(res, nd, B, monkeypatch):
    """The stride-2 input gradient as ONE launch over the four output-parity classes (b3d_conv_opts.nclass) against four
    launches: the same taps per output pixel.  The merged launch has four times the work items, so the dispatcher may pick
    another kernel variant (stacked tiles / row window) whose K loop runs in another order: fp32 summation-order differences
    only, 2e-5 of the largest magnitude on the input gradients (they pass through input-gradient kernels only)."""
    import b3d.conv as b3d_conv
    from models import gan
    args = GC.make_args(res, nd)
    _, D = GC.build(gan, args)
    D.cuda().train()
    z, c, alpha, tex, mesh = [t.cuda() for t in GC.inputs(args, B=B)]
    x0 = torch.cat((tex, alpha), dim=1)
    saved = {n: b.clone() for n, b in D.named_buffers()}
    got = []
    for per_class in (True, False):
        if per_class:
            monkeypatch.setattr(b3d_conv, "_merge_parity_classes", lambda classes: False)
        else:
            monkeypatch.undo()
        with torch.no_grad():
            for n, b in D.named_buffers():
                b.copy_(saved[n])
        D.zero_grad()
        x = x0.clone().requires_grad_(True)
        mm = mesh.clone().requires_grad_(True)
        out, _ = D(x, mm, c)
        g = torch.Generator(device="cuda").manual_seed(3)
        sum((o * torch.randn(o.shape, device=o.device, generator=g)).sum() for o in out).backward()
        torch.cuda.synchronize()
        got.append((x.grad.clone(), mm.grad.clone()))
    _close(got[1][0], got[0][0], 2e-5, "input gradient")
    _close(got[1][1], got[0][1], 2e-5, "mesh-map gradient")
