"""Weight gradient (b3d_conv2d_wgrad_tf32) at the edges of its pipeline, on every kernel instance, against the fp64
reference of tests/test_wgrad_regA_gpu.py (which covers cfg3's geometries).

The consumers keep one wgmma group in flight: a slice's dY fragments load into one of two register sets while the previous
slice's group runs, the loop takes two slices per turn, and the raw-input stem's two consumer warpgroups take alternate
slices.  So the cases run CTAs with 1, 2, 3 and an odd number of K slices, and a stem launch whose second consumer
warpgroup gets no slice.  wgrad_splits gives every CTA at least 8 slices once it splits K, so the short CTAs come from
launches of few slices (one split), and a split launch (17 slices over 2 CTAs: 8 and 9) covers an odd count behind a split.
Each case runs both dW layouts, the tap-major one with dY read through a row pitch wider than Wout and X from column 1 of a
wider buffer, and a one-split launch is repeated to show it is bitwise deterministic.

The producer's transpose of the raw X slice into the K-major B tiles (csrc/tc_conv.cu: xt_chunk, xt_src_offset,
xt_dst_offset) is checked on the CPU for coverage and bank conflicts."""
import ctypes

import pytest
import torch

import conv_plan as P
from test_wgrad_regA_gpu import _ref_wgrad

TOL = 4e-3


# mirrors of the device functions in csrc/tc_conv.cu
def xt_chunk(i):
    return (((i & 7) >> 1) ^ ((i >> 4) & 3)) | (((i >> 3) & 1) << 2)


def xt_src_offset(i, px, wrows):
    return ((i >> 6) * wrows + px) * 128 + (i & 7) * 16


def xt_dst_offset(i, j):
    return ((i >> 6) * 32 + 4 * (i & 7) + j) * 128 + ((xt_chunk(i) ^ ((4 * (i & 7) + j) & 7)) << 4)


@pytest.mark.parametrize("BN,T", [(64, 1), (128, 1), (64, 2), (128, 2), (64, 3)])
def test_x_transpose_covers_the_tiles_without_bank_conflicts(BN, T):
    """Tap t's tile gets B[ci][k] = window[k + t][ci] for every channel row and K index exactly once, in the 128-byte
    swizzle desc_k128 reads; each quarter warp's 16-byte loads and stores hit eight different bank groups."""
    wrows = 32 if T == 1 else 36
    tiles = [dict() for _ in range(T)]
    tasks = 2 * BN
    for i in range(tasks):
        q = xt_chunk(i)
        for t in range(T):
            for j in range(4):
                d = xt_dst_offset(i, j)
                assert d % 16 == 0 and 0 <= d < BN * 128
                for e in range(4):                           # element e of the stored float4: window pixel 4q + t + e
                    src = xt_src_offset(i, 4 * q + t + e, wrows) + 4 * j
                    assert 4 * q + t + e < wrows
                    blk, px, ch = src // (wrows * 128), src // 128 % wrows, src % 128 // 4
                    ci, k = d // 128, 4 * ((d // 16 % 8) ^ (d // 128 % 8)) + e
                    assert (blk * 32 + ch, px) == (ci, k + t)
                    assert (ci, k) not in tiles[t]
                    tiles[t][(ci, k)] = True
    for t in range(T):
        assert len(tiles[t]) == BN * 32
    for i0 in range(0, tasks, 8):                               # a quarter warp: eight consecutive tasks
        quarter = range(i0, i0 + 8)
        for u in range(T + 3):
            assert len({xt_src_offset(i, 4 * xt_chunk(i) + u, wrows) // 16 % 8 for i in quarter}) == 8
        for j in range(4):
            assert len({xt_dst_offset(i, j) // 16 % 8 for i in quarter}) == 8


# name, N, Cin, H, W, Cout, kh, kw, pad_y, stride — K slices per CTA in the comment
CASES = [
    ("t1_bn64_k1", 1, 64, 4, 6, 128, 3, 3, 1, 1),               # Wout 4: one 4 x 8 pixel box, 1 slice
    ("t1_bn64_k2", 2, 64, 4, 6, 128, 3, 3, 1, 1),               # 2
    ("t1_bn64_k3", 3, 64, 4, 6, 128, 3, 3, 1, 1),               # 3
    ("t1_bn128_k1", 1, 128, 4, 6, 128, 3, 3, 1, 1),
    ("t1_bn128_k5", 5, 128, 4, 6, 256, 3, 3, 1, 1),
    ("t3_k1", 1, 64, 1, 34, 64, 3, 3, 1, 1),                    # Wout 32, one row: 1 slice
    ("t3_k2", 2, 64, 1, 34, 64, 3, 3, 1, 1),
    ("t3_k3", 3, 64, 1, 34, 64, 3, 3, 1, 1),
    ("t3_split_8_9", 17, 64, 1, 34, 64, 3, 3, 1, 1),            # 17 slices over 2 splits
    ("t2_bn64_k1", 1, 64, 2, 66, 128, 4, 4, 1, 2),              # stride 2, Wout 32, Hout 1
    ("t2_bn64_k3", 3, 64, 2, 66, 128, 4, 4, 1, 2),
    ("t2_bn128_k1", 1, 128, 2, 66, 256, 4, 4, 1, 2),
    ("t2_bn128_k2", 2, 128, 2, 66, 256, 4, 4, 1, 2),
    ("t2_bn128_k3", 3, 128, 2, 66, 256, 4, 4, 1, 2),
    ("t2_bn128_split", 9, 128, 4, 66, 256, 4, 4, 1, 2),         # Hout 2: 18 slices
]


def _launch(dy, x, dw, N, H, W, Cin, Hout, Wout, Cout, kh, kw, pad_y, st, x_off, tap_major, pitch):
    from b3d import check, lib, ptr, stream_ptr
    check(lib.b3d_conv2d_wgrad_tf32(ctypes.c_void_p(dy.data_ptr()), ptr(x), ptr(dw), N, H, W, Cin, Hout, Wout, Cout, kh, kw,
                                    pad_y, st, x_off, tap_major, 0, pitch, stream_ptr(x)))


@pytest.mark.gpu
@pytest.mark.parametrize("name,N,Cin,H,W,Cout,kh,kw,pad_y,st", CASES, ids=[c[0] for c in CASES])
def test_wgrad_pipeline_edges(name, N, Cin, H, W, Cout, kh, kw, pad_y, st):
    from b3d import last_variant
    dev = "cuda:0"
    Hout, Wout = (H + 2 * pad_y - kh) // st + 1, (W - kw) // st + 1
    (plan,) = P.wgrad_tf32(N, H, W, Cin, Cout, kh, kw, pad_y, st, sms=torch.cuda.get_device_properties(0).multi_processor_count)
    g = torch.Generator(device=dev).manual_seed(N * 1000 + Cin + Cout + W)
    pitch = Wout + 3
    xwide = torch.randn(N, H, W + 2, Cin, device=dev, generator=g)
    dywide = torch.randn(N, Hout, pitch, Cout, device=dev, generator=g)
    x, dy = xwide[:, :, 1:W + 1].contiguous(), dywide[:, :, :Wout].contiguous()
    ref = _ref_wgrad(dy, x, kh, kw, pad_y, st)
    scale = float(ref.abs().max())

    a = torch.zeros(Cout, Cin, kh, kw, device=dev)
    _launch(dy, x, a, N, H, W, Cin, Hout, Wout, Cout, kh, kw, pad_y, st, 0, 0, 0)
    assert last_variant() == plan.instance, (name, last_variant(), plan)
    b = torch.zeros(kh * kw, Cout, Cin, device=dev)
    _launch(dywide, xwide, b, N, H, W + 2, Cin, Hout, Wout, Cout, kh, kw, pad_y, st, 1, 1, pitch)
    torch.cuda.synchronize()
    err_a = float((a.double().permute(2, 3, 0, 1).reshape(kh * kw, Cout, Cin) - ref).abs().max())
    err_b = float((b.double() - ref).abs().max())
    assert err_a <= TOL * scale, (name, plan.kslices, plan.splits, "[Cout][Cin][kh][kw]", err_a, scale)
    assert err_b <= TOL * scale, (name, plan.kslices, plan.splits, "tap-major, dy_row_pitch, x_off", err_b, scale)
    if plan.splits == 1:
        b2 = torch.zeros_like(b)
        _launch(dywide, xwide, b2, N, H, W + 2, Cin, Hout, Wout, Cout, kh, kw, pad_y, st, 1, 1, pitch)
        torch.cuda.synchronize()
        assert torch.equal(b, b2), name
    else:
        assert plan.kslices % plan.splits != 0 or (plan.kslices // plan.splits) % 2 == 1, plan


# raw-input stem: N, H, W (x-padded), Cout — Hout = H (pad_y 2), Wout = W - 4, one 32-pixel segment per row
STEM = [("stem_k1", 1, 1, 36, 64), ("stem_k2", 1, 2, 36, 64), ("stem_k3", 3, 1, 36, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,N,H,W,Cout", STEM, ids=[c[0] for c in STEM])
def test_wgrad_stem_pipeline_edges(name, N, H, W, Cout):
    """1 slice (the second consumer warpgroup has none), 2 (one each) and 3 (two for the first)."""
    from b3d import check, last_variant, lib, ptr, stream_ptr
    dev, kw, fold_kh, pad_y, cf = "cuda:0", 5, 5, 2, 64
    Hout, Wout = H + 2 * pad_y - fold_kh + 1, W - kw + 1
    (plan,) = P.wgrad(N, H, W, 8, Cout, 1, kw, pad_y, 1, fold_kh=fold_kh, fold_cin=cf)
    assert plan.splits == 1 and plan.kslices == N * H
    g = torch.Generator(device=dev).manual_seed(N * 31 + H)
    x = torch.randn(N, H, W, 8, device=dev, generator=g)
    dy = torch.randn(N, Hout, Wout, Cout, device=dev, generator=g)
    xp = torch.nn.functional.pad(x.double(), (0, 0, 0, 0, pad_y, pad_y))
    d = dy.double().reshape(-1, Cout).t()
    ref = torch.zeros(kw, Cout, cf, dtype=torch.float64, device=dev)
    for r in range(fold_kh):
        for s in range(kw):
            ref[s, :, 8 * r:8 * r + 8] = d @ xp[:, r:r + Hout, s:s + Wout].reshape(-1, 8)
    outs = []
    for _ in range(2):
        tm = torch.zeros(kw, Cout, cf, device=dev)
        check(lib.b3d_conv2d_wgrad_tf32(ptr(dy), ptr(x), ptr(tm), N, H, W, cf, Hout, Wout, Cout, 1, kw, pad_y, 1, 0, 1, fold_kh, 0,
                                        stream_ptr(x)))
        assert last_variant() == plan.instance, last_variant()
        outs.append(tm)
    torch.cuda.synchronize()
    err = float((outs[0].double() - ref).abs().max())
    assert err <= TOL * float(ref.abs().max()), (name, err)
    assert torch.equal(outs[0], outs[1]), name
