"""Masked input gradients whose mask tile the producer loads with TMA into the operand ring (b3d_conv_opts.mask): the cases
where that path has behaviour of its own, against the same fp64 reference and tolerances as test_dgrad_mask_gpu.py.

- 256-wide tiles: 8 mask chunks per item wrap the 4-stage ring, over CTAs that take one or two items;
- 64-wide tiles (each consumer warpgroup owns alternate items): CTAs with three items (an odd count) next to CTAs with
  two, and a strip launch with fewer items than SMs;
- tiles that overhang the mask tensor in H and in N, so part of the box is TMA's zero fill;
- the host's refusal of a mask TMA cannot describe (a base that is not 16-byte aligned, OC % 4 != 0)."""
import pytest
import torch

from test_dgrad_mask_gpu import DEV, SLOPE, _check, _run

pytestmark = pytest.mark.gpu

# name, Cin (channels of gx and of the mask), H, W (x-padded input), Cout, k, pad_y, stride, N, instances that must run
GEOM = [
    # 6 x 30 rows of 128-pixel tiles (180 items on 132 SMs) + a 2-column strip of 2 x 16 x 4 tiles: rows 30, 31 and images
    # 6, 7 of its second tiles lie outside the tensor
    ("256.ring_wrap", 256, 30, 130, 64, 3, 1, 1, 6, {"conv_wgmma<256,4>"}),
    # 2 x 165 row tiles = 330 items: 66 CTAs take three, 66 take two; the strip's 2 x 64 x 1 tiles make 6 items, rows
    # 165 .. 191 outside the tensor
    ("64.odd_items", 64, 165, 130, 64, 3, 1, 1, 2, {"conv_wgmma_rowwin<64,3,4>", "conv_wgmma<64,8>"}),
    # 5 images of 6 x 10: 8 x 4 x 4 tiles (8 items), overhanging in x, H (rows 6, 7) and N (images 5 .. 7)
    ("64.overhang", 64, 6, 10, 64, 3, 1, 1, 5, {"conv_wgmma<64,8>"}),
    ("128.overhang", 128, 6, 10, 64, 3, 1, 1, 5, {"conv_wgmma<128,6>"}),
]


@pytest.mark.parametrize("sums", [False, True])
@pytest.mark.parametrize("name,Cin,H,W,Cout,k,pad_y,stride,N,need", GEOM, ids=[c[0] for c in GEOM])
def test_masked_input_gradient_tma_edges(name, Cin, H, W, Cout, k, pad_y, stride, N, need, sums):
    gx, r, st, ran = _run(N, Cin, H, W, Cout, k, pad_y, stride, sums=sums, pitched=False, seed=sum(map(ord, name)) + sums)
    assert need == ran, (name, sorted(ran))
    _check(gx, r, st, name)


def _launch(mask, Cin):
    import b3d.conv as C
    N, H, W, Cout = 2, 8, 130, 64
    g = torch.Generator().manual_seed(7)
    wd = C._d_layout((torch.randn(9, Cout, Cin, generator=g) * 0.05).to(DEV))
    gy = torch.randn(N, H, W - 2, Cout, generator=g).to(DEV)
    return C._dgrad(gy, wd, (H, W), 3, 3, 1, 1, mask=mask(N, H, W), slope=SLOPE)


def test_mask_tma_refusals():
    from b3d import B3DError
    Cin = 64
    n = 2 * 8 * 130 * Cin
    shifted = torch.randn(n + 1, device=DEV)[1:]                  # 4 bytes past a 16-byte boundary
    with pytest.raises(B3DError, match="16-byte aligned"):
        _launch(lambda N, H, W: shifted.view(N, H, W, Cin), Cin)
    with pytest.raises(B3DError, match="OC % 4 == 0"):
        _launch(lambda N, H, W: torch.randn(N, H, W, 6, device=DEV), 6)
    # the same launch with an aligned mask of 64 channels runs
    gx = _launch(lambda N, H, W: torch.randn(N, H, W, Cin, device=DEV), Cin)
    assert bool(torch.isfinite(gx).all())
