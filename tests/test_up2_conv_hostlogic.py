"""The upsampled-input convolution of the generator (b3d/conv.py: conv2d_up2_banked) as index arithmetic, in fp64 on the CPU.

conv3x3(pad_x(up2(X), 1), W, padding=(1, 0)) is computed as a stride-2 transposed convolution of Xp = pad_x(X, 1) with
the phase weights P (csrc/sn_kernels.cu), its input gradient as a 4x4 stride-2 correlation of dY on D4, and its weight
gradient as dP^T from three column launches folded back to the nine taps.  Here each launch the helpers describe
(up2_fprop_taps, up2_dgrad_taps, up2_wgrad_columns) is emulated tap by tap and checked against torch's F.interpolate +
F.conv2d and its autograd, for replicate and circular x padding, odd and even sizes and one-row maps."""
import pytest
import torch
import torch.nn.functional as F

import b3d.conv as C

A = [[[1, 0, 0], [0, 1, 1]], [[1, 1, 0], [0, 0, 1]]]          # A_p[a][k] (csrc/sn_kernels.cu)


def phase_weights(w):
    """w [Cout,Cin,3,3] -> P [16][Cout][Cin] as the bank writes it (without the tf32 rounding)."""
    P = torch.zeros(16, *w.shape[:2], dtype=w.dtype)
    for py in range(2):
        for px in range(2):
            for a in range(2):
                for b in range(2):
                    q = ((py * 2 + px) * 2 + a) * 2 + b
                    for k in range(3):
                        for l in range(3):
                            if A[py][a][k] and A[px][b][l]:
                                P[q] += w[:, :, k, l]
    return P


def d4_layout(P):
    """P [16][Cout][Cin] -> D4 [16][Cin][Cout]: tap (r, s) = (3 - py - 2a, 3 - px - 2b) carries P[q]^T."""
    D4 = torch.zeros(16, P.shape[2], P.shape[1], dtype=P.dtype)
    for q in range(16):
        py, px, a, b = q >> 3, (q >> 2) & 1, (q >> 1) & 1, q & 1
        D4[(3 - py - 2 * a) * 4 + 3 - px - 2 * b] = P[q].t()
    return D4


def fold(dpt):
    """dP^T [16][Cin][Cout] (D4's tap order) -> dW [Cout,Cin,3,3], the adjoint of phase_weights (b3d_up2_fold)."""
    Cin, Cout = dpt.shape[1:]
    dw = torch.zeros(Cout, Cin, 3, 3, dtype=dpt.dtype)
    for q in range(16):
        py, px, a, b = q >> 3, (q >> 2) & 1, (q >> 1) & 1, q & 1
        g = dpt[(3 - py - 2 * a) * 4 + 3 - px - 2 * b].t()
        for k in range(3):
            for l in range(3):
                if A[py][a][k] and A[px][b][l]:
                    dw[:, :, k, l] += g
    return dw


def shifted(x, dy, dx, Hout, Wout, sy=1, sx=1):
    """x [N,C,H,W] read at (sy*i + dy, sx*j + dx) for i < Hout, j < Wout, zero outside (the kernels' TMA fill)."""
    N, Cc, H, W = x.shape
    out = torch.zeros(N, Cc, Hout, Wout, dtype=x.dtype)
    for i in range(Hout):
        yi = sy * i + dy
        if not 0 <= yi < H:
            continue
        for j in range(Wout):
            xj = sx * j + dx
            if 0 <= xj < W:
                out[:, :, i, j] = x[:, :, yi, xj]
    return out


def pad_x(x, mode):
    return torch.cat([x[..., :1], x, x[..., -1:]], -1) if mode == "replicate" else torch.cat([x[..., -1:], x, x[..., :1]], -1)


def reference(xp, w):
    """conv3x3(pad_x(up2(X), 1), w, padding=(1, 0)) from Xp = pad_x(X, 1): the pad columns of the upsampled map are
    Xp's pad columns, its interior the upsampled interior of Xp."""
    u = F.interpolate(xp[..., 1:-1], scale_factor=2, mode="nearest")
    return F.conv2d(torch.cat([xp[..., :1].repeat_interleave(2, 2), u, xp[..., -1:].repeat_interleave(2, 2)], -1), w, padding=(1, 0))


def up_forward(xp, P):
    N, _, H, Wp = xp.shape
    W = Wp - 2
    y = torch.zeros(N, P.shape[1], 2 * H, 2 * W, dtype=xp.dtype)
    dy, dx, wtap, cls = C.up2_fprop_taps()
    for c, (py, px) in enumerate(cls):
        for t in range(4 * c, 4 * c + 4):
            y[:, :, py::2, px::2] += torch.einsum("oc,nchw->nohw", P[wtap[t]], shifted(xp, dy[t], dx[t], H, W))
    return y


def up_dgrad(gy, D4):
    N, _, H2, W2 = gy.shape
    H, Wp = H2 // 2, W2 // 2 + 2
    dy, dx = C.up2_dgrad_taps()
    return sum(torch.einsum("co,nohw->nchw", D4[t], shifted(gy, dy[t], dx[t], H, Wp, 2, 2)) for t in range(16))


def up_wgrad(gy, xp):
    """dP^T [16][Cin][Cout] as the three swapped-role weight-gradient launches compute it."""
    N, Cin, H, Wp = xp.shape
    dpt = torch.zeros(16, Cin, gy.shape[1], dtype=xp.dtype)
    for j0, w, x_off in C.up2_wgrad_columns(Wp - 2):
        xs = xp[..., j0:j0 + w]
        for r in range(4):
            for s in range(4):
                dpt[r * 4 + s] += torch.einsum("nchw,nohw->co", xs, shifted(gy, r - 1, s + x_off, H, w, 2, 2))
    return dpt


@pytest.mark.parametrize("mode", ["replicate", "circular"])
@pytest.mark.parametrize("H,W", [(1, 1), (1, 4), (2, 3), (3, 2), (4, 5)])
def test_up2_identity(mode, H, W):
    g = torch.Generator().manual_seed(H * 10 + W)
    N, Cin, Cout = 2, 3, 4
    x = torch.randn(N, Cin, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Cout, Cin, 3, 3, generator=g, dtype=torch.float64, requires_grad=True)
    xp = pad_x(x, mode).requires_grad_(True)
    ref = reference(xp, w)
    # the reference is the generator's own upsample -> pad -> conv of the unfused path
    assert torch.allclose(ref, F.conv2d(pad_x(F.interpolate(x, scale_factor=2, mode="nearest"), mode), w, padding=(1, 0)))
    P = phase_weights(w.detach())
    y = up_forward(xp.detach(), P)
    assert torch.allclose(y, ref, atol=1e-12, rtol=0)
    gy = torch.randn(ref.shape, generator=g, dtype=torch.float64)
    gxp, gw = torch.autograd.grad(ref, (xp, w), gy)
    assert torch.allclose(up_dgrad(gy, d4_layout(P)), gxp, atol=1e-12, rtol=0)
    assert torch.allclose(fold(up_wgrad(gy, xp.detach())), gw, atol=1e-12, rtol=0)


def test_up2_tap_lists():
    dy, dx, wtap, cls = C.up2_fprop_taps()
    assert cls == [(0, 0), (0, 1), (1, 0), (1, 1)]
    assert wtap == list(range(16))                     # P is written in class-major tap order
    assert dy[:4] == [-1, -1, 0, 0] and dx[:4] == [0, 1, 0, 1] and dy[12:] == [0, 0, 1, 1] and dx[12:] == [1, 2, 1, 2]
    ddy, ddx = C.up2_dgrad_taps()
    assert sorted(set(ddy)) == [-1, 0, 1, 2] and sorted(set(ddx)) == [-3, -2, -1, 0]
    assert C.up2_wgrad_columns(64) == [(1, 64, -1), (0, 1, -3), (65, 1, 127)]
