"""Plain-torch restatement of the fused batch-norm glue (b3d.ew.cbn_act_pad / bn_act_pad) for the GPU tests: run in fp64
it is the reference, run in fp32 it measures how much fp32 arithmetic alone moves the result."""
import types

import torch
import torch.nn.functional as F

EPS = 1e-5
EMB = 32


def ref_glue(y, g, b, skip=None, off=0, up=1, pad=1, post=False, slope=0.2, run=None, eps=EPS, clamp=False):
    """y [N,C,H,W]; g, b [N or 1, C] (gamma, beta rows: per sample for CBN, one shared row for BNAffine); run = (running mean,
    running var) in eval mode, None for batch statistics; clamp = the SyncBN formula inv_std = clamp(var, eps)^-1/2.
    -> (out, pre = input of the first activation, mid = input of the second, mean, biased variance)."""
    W = y.shape[3]
    if run is None:
        m = y.mean(dim=(0, 2, 3))
        v = y.var(dim=(0, 2, 3), unbiased=False)
        inv = v.clamp(min=eps).rsqrt() if clamp else (v + eps).rsqrt()
    else:
        m, v = (t.to(y.dtype) for t in run)
        inv = (v + eps).rsqrt()
    pre = (y - m[None, :, None, None]) * inv[None, :, None, None] * (1 + g[:, :, None, None]) + b[:, :, None, None]
    h = F.leaky_relu(pre, slope)
    if skip is not None:
        h = h + skip[..., off:off + W]
    mid = h
    if post:
        h = F.leaky_relu(h, slope)
    if up == 2:
        h = F.interpolate(h, scale_factor=2, mode='nearest')
    if pad:
        h = F.pad(h, (pad, pad, 0, 0), mode='replicate')
    return h, pre, mid, m, v


def clear_kinks(y, g, b, skip=None, off=0, post=False, slope=0.2, run=None, clamp=False, thr=1e-4):
    """Corrections (dy, dskip) in fp64 that move the rare elements whose activation input lies within `thr` of the kink
    4*thr away from it.  There fp32 and fp64 may take different branches, and the derivative jumps by (1 - slope): a
    difference of definition, not of accuracy.  The statistics move by ~thr / count, far less than thr."""
    with torch.no_grad():
        _, pre, _, m, v = ref_glue(y, g, b, run=run, clamp=clamp, pad=0, slope=slope)
        inv = v.clamp(min=EPS).rsqrt() if clamp and run is None else (v + EPS).rsqrt()
        a = inv[None, :, None, None] * (1 + g[:, :, None, None])            # d pre / d y
        sgn = torch.where(pre >= 0, 1.0, -1.0).to(y.dtype)
        dy = torch.where(pre.abs() < thr, sgn * 4 * thr / a, torch.zeros_like(pre))
        dskip = None
        if skip is not None and post:
            W = y.shape[3]
            mid = F.leaky_relu(pre + a * dy, slope) + skip[..., off:off + W]
            ds = torch.where(mid.abs() < thr, torch.where(mid >= 0, 1.0, -1.0).to(y.dtype) * 4 * thr, torch.zeros_like(mid))
            dskip = torch.zeros_like(skip)
            dskip[..., off:off + W] = ds
    return dy, dskip


def make_cbn(C, seed, norm_g='batch', **bn_kw):
    """models.gan.ConditionalBatchNorm2d with gamma / beta of a useful size (std ~0.3 per sample) and per-channel running
    statistics away from (0, 1)."""
    from models.gan import ConditionalBatchNorm2d
    torch.manual_seed(seed)
    m = ConditionalBatchNorm2d(types.SimpleNamespace(norm_g=norm_g), C, EMB)
    if bn_kw:
        m.norm = type(m.norm)(C, affine=False, **bn_kw)
    with torch.no_grad():
        for lin in (m.fc_gamma, m.fc_beta):
            lin.weight.normal_(0.0, 0.3 / EMB ** 0.5)
            lin.bias.normal_(0.0, 0.1)
        if m.norm.running_mean is not None:
            m.norm.running_mean.normal_(0.0, 0.5)
            m.norm.running_var.uniform_(0.5, 2.0)
    return m


def make_bn(C, seed, **bn_kw):
    """torch.nn.BatchNorm2d (the reconstruction network's norm) with weight / bias away from (1, 0)."""
    torch.manual_seed(seed)
    m = torch.nn.BatchNorm2d(C, **bn_kw)
    with torch.no_grad():
        m.weight.uniform_(0.6, 1.4)
        m.bias.normal_(0.0, 0.2)
        if m.running_mean is not None:
            m.running_mean.normal_(0.0, 0.5)
            m.running_var.uniform_(0.5, 2.0)
    return m


def errors(got, r64, r32, mask=None):
    """(max |got - fp64|, max |fp32 torch - fp64|, max |fp64|) over `mask` (all elements if None)."""
    got, r64, r32 = got.detach().double(), r64.detach().double(), r32.detach().double()
    if mask is not None:
        got, r64, r32 = got[mask], r64[mask], r32[mask]
    return float((got - r64).abs().max()), float((r32 - r64).abs().max()), float(r64.abs().max())


def assert_close(name, got, r64, r32, ceiling, mask=None):
    """|kernel - fp64| <= 4 |torch fp32 - fp64| + 1e-6 max|fp64|, and never above `ceiling` * max|fp64|."""
    assert got.shape == r64.shape, f"{name}: shape {tuple(got.shape)} != {tuple(r64.shape)}"
    err, gap, scale = errors(got, r64, r32, mask)
    tol = 4.0 * gap + 1e-6 * scale
    print(f"  {name:28s} err/max {err / max(scale, 1e-30):.2e}  fp32-gap/max {gap / max(scale, 1e-30):.2e}  err/gap "
          f"{err / max(gap, 1e-30):.2f}")
    assert err <= tol, f"{name}: |kernel - fp64| = {err:.3e} > 4 x fp32 gap {gap:.3e} + 1e-6 x {scale:.3e}"
    assert err <= ceiling * scale, f"{name}: |kernel - fp64| = {err:.3e} > {ceiling:g} x max {scale:.3e}"
