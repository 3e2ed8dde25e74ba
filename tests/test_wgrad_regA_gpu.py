"""Weight gradient (b3d_conv2d_wgrad_tf32) at the benchmark's cfg3 conv geometries, batch 32 for the generator's layers and
64 for the discriminator's (tools/time_convs.py), against an fp64 reference: per tap, dY^T @ X_shifted as a float64 GEMM.
Each geometry runs twice: the [Cout][Cin][kh][kw] layout from dense operands, and the tap-major layout with dY read through
a row pitch wider than Wout and X read from column x_off = 1 of a wider buffer (the extra columns hold random values, so a
wrong offset shows).  Tolerance as tests/test_conv_gpu.py: max |err| <= 4e-3 max |ref|.

The kernel feeds dY to wgmma from registers, loaded straight from the TMA-staged, 128-byte swizzled dY tile; the CPU test
checks the address function of those loads (csrc/tc_conv.cu: wgrad_row_co, dy_tile_offset) for bank conflicts and coverage."""
import ctypes

import pytest
import torch

import conv_plan as P

TOL = 4e-3
B = 32
# name, N, Cin, H, W (x-padded), Cout, k, pad_y, stride — the weight-gradient launches of one cfg3 step
CFG3 = [("G.blk1.conv", B, 512, 8, 6, 512, 3, 1, 1), ("G.blk2.conv1", B, 512, 16, 10, 256, 3, 1, 1),
        ("G.blk3a.conv", B, 256, 32, 18, 256, 3, 1, 1), ("G.blk4.conv1", B, 256, 64, 34, 128, 3, 1, 1),
        ("G.blk4.conv2", B, 128, 64, 34, 128, 3, 1, 1), ("G.blk5.conv", B, 128, 128, 66, 128, 3, 1, 1),
        ("G.blk6.conv1", B, 128, 256, 130, 64, 3, 1, 1), ("G.blk6.conv2", B, 64, 256, 130, 64, 3, 1, 1),
        ("G.blk6.short", B, 128, 256, 128, 64, 1, 0, 1), ("G.conv_final", B, 64, 256, 132, 3, 5, 2, 1),
        ("D1.c1.kwfold", 2 * B, 64, 256, 256, 64, (5, 1), 2, 1), ("D1.c1.khfold", 2 * B, 64, 256, 260, 64, (1, 5), 0, 1),
        ("D1.conv2", 2 * B, 64, 256, 258, 128, 4, 1, 2), ("D1.conv3", 2 * B, 128, 128, 130, 256, 4, 1, 2),
        ("D1.conv4", 2 * B, 256, 64, 66, 512, 4, 1, 2), ("D1.conv5", 2 * B, 512, 32, 36, 1, 5, 2, 1)]


def _kh_kw(k):
    return k if isinstance(k, tuple) else (k, k)


def _out_size(H, W, kh, kw, pad_y, st):
    return (H + 2 * pad_y - kh) // st + 1, (W - kw) // st + 1


def test_cfg3_has_a_ragged_k_split():
    """On an H100 SXM (132 SMs) the K slices of some geometries do not divide evenly among the splits wgrad_splits picks
    (the k_lo / k_hi rounding of the kernel is exercised)."""
    ragged = []
    for _, N, Cin, H, W, Cout, k, py, st in CFG3:
        kh, kw = _kh_kw(k)
        (launch,) = P.wgrad_tf32(N, H, W, Cin, -(-Cout // 32) * 32, kh, kw, py, st, sms=132)
        ragged.append(launch.kslices % launch.splits != 0)
    assert any(ragged)


# mirrors of the device functions in csrc/tc_conv.cu
def wgrad_row_co(m):
    return (m & 35) | ((m & 8) >> 1) | ((m & 16) >> 1) | ((m & 4) << 2)


def dy_tile_offset(co, px):
    return (co >> 5) * 4096 + px * 128 + ((((co >> 2) & 7) ^ (px & 7)) << 4) + (co & 3) * 4


def test_dy_fragment_loads_are_conflict_free_and_cover_the_tile():
    """Every fragment load (consumer warpgroup h, warp w, register e, K step k) hits 32 different banks; the m64k8 fragment
    of each warpgroup holds every (row, k) exactly once; over both warpgroups and the four K steps every dY[co][px] of the
    128 x 32 slice is read exactly once."""
    assert sorted(wgrad_row_co(m) for m in range(64)) == list(range(64))
    read = {}
    for h in range(2):
        frag = set()
        for w in range(4):
            for e in range(4):
                for k in range(4):
                    banks = set()
                    for lane in range(32):
                        m, kc = 16 * w + lane // 4 + 8 * (e & 1), lane % 4 + 4 * (e >> 1)
                        if k == 0:
                            frag.add((m, kc))
                        co, px = h * 64 + wgrad_row_co(m), 8 * k + kc
                        off = dy_tile_offset(co, px)
                        assert off % 4 == 0 and 0 <= off < 128 * 32 * 4
                        banks.add(off // 4 % 32)
                        read[(co, px)] = read.get((co, px), 0) + 1
                        assert off == dy_tile_offset(co, 8 * k + kc % 8) and off - dy_tile_offset(co, kc) == 1024 * k
                    assert len(banks) == 32, (h, w, e, k)
        assert frag == {(m, kc) for m in range(64) for kc in range(8)}
    assert len(read) == 128 * 32 and set(read.values()) == {1}
    assert len({dy_tile_offset(co, px) for co, px in read}) == 128 * 32


def _ref_wgrad(dy, x, kh, kw, pad_y, st):
    """dW [kh*kw, Cout, Cin] in float64: per tap, dY^T @ X shifted by the tap (zero rows above / below = pad_y)."""
    N, Hout, Wout, Cout = dy.shape
    xp = torch.nn.functional.pad(x.double(), (0, 0, 0, 0, pad_y, pad_y))
    d = dy.double().reshape(-1, Cout)
    out = []
    for r in range(kh):
        for s in range(kw):
            xs = xp[:, r:r + st * (Hout - 1) + 1:st, s:s + st * (Wout - 1) + 1:st]
            out.append(d.t() @ xs.reshape(-1, x.shape[3]))
    return torch.stack(out)


@pytest.mark.gpu
@pytest.mark.parametrize("name,N,Cin,H,W,Cout,k,pad_y,st", CFG3, ids=[c[0] for c in CFG3])
def test_wgrad_cfg3_geometry(name, N, Cin, H, W, Cout, k, pad_y, st):
    from b3d import check, last_variant, lib, ptr, stream_ptr
    dev = "cuda:0"
    kh, kw = _kh_kw(k)
    Cout = -(-Cout // 32) * 32                     # the channel padding b3d.conv applies to thin heads
    Hout, Wout = _out_size(H, W, kh, kw, pad_y, st)
    g = torch.Generator(device=dev).manual_seed(Cin * 7 + Cout + kh)
    pitch = Wout + 3
    xwide = torch.randn(N, H, W + 2, Cin, device=dev, generator=g)
    dywide = torch.randn(N, Hout, pitch, Cout, device=dev, generator=g)
    x, dy = xwide[:, :, 1:W + 1].contiguous(), dywide[:, :, :Wout].contiguous()
    ref = _ref_wgrad(dy, x, kh, kw, pad_y, st)
    scale = float(ref.abs().max())

    a = torch.zeros(Cout, Cin, kh, kw, device=dev)
    check(lib.b3d_conv2d_wgrad_tf32(ptr(dy), ptr(x), ptr(a), N, H, W, Cin, Hout, Wout, Cout, kh, kw, pad_y, st, 0, 0, 0, 0,
                                    stream_ptr(x)))
    (plan,) = P.wgrad_tf32(N, H, W, Cin, Cout, kh, kw, pad_y, st, sms=torch.cuda.get_device_properties(0).multi_processor_count)
    assert last_variant() == plan.instance, (name, last_variant(), plan)
    b = torch.zeros(kh * kw, Cout, Cin, device=dev)
    check(lib.b3d_conv2d_wgrad_tf32(ctypes.c_void_p(dywide.data_ptr()), ptr(xwide), ptr(b), N, H, W + 2, Cin, Hout, Wout, Cout,
                                    kh, kw, pad_y, st, 1, 1, 0, pitch, stream_ptr(x)))
    torch.cuda.synchronize()
    err_a = float((a.double().permute(2, 3, 0, 1).reshape(kh * kw, Cout, Cin) - ref).abs().max())
    err_b = float((b.double() - ref).abs().max())
    assert err_a <= TOL * scale, (name, "[Cout][Cin][kh][kw]", err_a, scale)
    assert err_b <= TOL * scale, (name, "tap-major, dy_row_pitch, x_off", err_b, scale)
