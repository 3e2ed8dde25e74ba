"""Host checks of the harness behind tests/test_mesh_raster_fp64_gpu.py: oracle/mesh.py's decision record, the fp64
oracle's adjoint with the decisions pinned, stable_pixels on hand-built near-ties and the fp32 restatement of the CUDA
rasteriser's tile binning.  No GPU needed."""
import os
import tempfile

import pytest
import torch

from oracle import mesh as M


@pytest.fixture(scope="module")
def sphere():
    path = M.write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16)
    return M.TemplateData(M.load_obj(path), path)


def posed(T, B, seed):
    g = torch.Generator().manual_seed(seed)
    mesh_map = torch.randn(B, 3, 32, 32, generator=g) * 0.05
    q = torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=-1)
    s = 0.5 + 0.3 * torch.rand(B, 1, generator=g)
    t = (torch.rand(B, 3, generator=g) - 0.5) * 0.3
    vtx = M.transform_vertices(M.get_vertex_positions(T, mesh_map), s, t, q)
    p3d, p2d, normal = M.ortho_projection(vtx, T.faces)
    attr = torch.rand(B, p2d.shape[1], 6, generator=g) * 2 - 1
    return p3d, p2d, normal[:, :, 2:3], attr


@pytest.mark.parametrize("dt", [torch.float32, torch.float64])
def test_record_leaves_outputs_bit_identical(sphere, dt):
    p3d, p2d, nz, attr = (t.to(dt) for t in posed(sphere, 2, 1))
    g = torch.Generator().manual_seed(2)
    w, wp = torch.rand(2, 40, 56, 2, generator=g).to(dt), torch.rand(2, 40, 56, 1, generator=g).to(dt)
    outs, grads = [], []
    for record in (None, {}):
        p, a = p2d.clone().requires_grad_(True), attr.clone().requires_grad_(True)
        o = M.rasterize(p3d, p, nz, a, 40, 56, record=record)
        outs.append(o)
        grads.append(torch.autograd.grad((o[0] * w).sum() + (o[1] * wp).sum(), [p, a]))
        if record is not None:
            assert torch.equal(record["imidx"], o[2]) and int(record["soft_n"].max()) > 0
    for x, y in zip(outs[0] + grads[0], outs[1] + grads[1]):
        assert torch.equal(x, y)


def tiny_scene():
    """Three faces on a 12 x 10 image: two overlapping front faces and one back face (soft silhouette only)."""
    p2d = torch.tensor([[[-0.55, -0.50, 0.30, -0.35, -0.20, 0.45],
                         [-0.10, -0.60, 0.62, 0.05, -0.35, 0.25],
                         [0.20, 0.55, 0.75, 0.70, 0.45, 0.95]]], dtype=torch.float64)
    z = torch.tensor([[[0.1, 0.2, 0.3], [0.4, -0.1, 0.0], [0.0, 0.1, 0.2]]], dtype=torch.float64)
    p3d = torch.stack([p2d[..., 0], p2d[..., 1], z[..., 0], p2d[..., 2], p2d[..., 3], z[..., 1],
                       p2d[..., 4], p2d[..., 5], z[..., 2]], dim=-1)
    nz = torch.tensor([[[1.0], [1.0], [-1.0]]], dtype=torch.float64)
    attr = torch.tensor([[[0.1, 0.9, 0.4, 0.7, -0.2, 0.3], [0.5, -0.5, 0.8, 0.2, 0.6, -0.9],
                          [0.3, 0.3, -0.4, 0.1, 0.9, 0.5]]], dtype=torch.float64)
    return p3d, p2d, nz, attr


def test_fp64_autograd_matches_finite_differences():
    """With every decision pinned (the record at +-h equals the record at the point), the fp64 oracle's gradient w.r.t.
    points2d and the attributes is the central difference of its forward, to 1e-6 relative."""
    p3d, p2d, nz, attr = tiny_scene()
    H, W = 12, 10
    kw = dict(delta=2000.0)                 # a soft silhouette that reaches a few pixels at this pitch
    r32, r64 = {}, {}
    M.rasterize(p3d.float(), p2d.float(), nz.float(), attr.float(), H, W, record=r32, **kw)
    M.rasterize(p3d, p2d, nz, attr, H, W, record=r64, **kw)
    stable = M.stable_pixels(r32, r64)
    assert bool((r64["imidx"] > 0).any()) and int(((r64["imidx"] == 0) & (r64["soft_n"] > 0) & stable).sum()) > 5
    g = torch.Generator().manual_seed(3)
    w = torch.rand(1, H, W, 2, generator=g, dtype=torch.float64) * stable.unsqueeze(-1)
    wp = torch.rand(1, H, W, 1, generator=g, dtype=torch.float64) * stable.unsqueeze(-1)

    def loss(p, a, rec=None):
        f, pr, _, _ = M.rasterize(p3d, p, nz, a, H, W, record=rec, **kw)
        return (f * w).sum() + (pr * wp).sum()

    p, a = p2d.clone().requires_grad_(True), attr.clone().requires_grad_(True)
    gp, ga = torch.autograd.grad(loss(p, a), [p, a])
    h = 1e-6
    keys = ("imidx", "soft_n", "soft_sig")
    for x, gx in ((p2d, gp), (attr, ga)):
        fd = torch.zeros_like(x)
        for i in range(x.numel()):
            vals = []
            for s in (1, -1):
                xs = x.clone().view(-1)
                xs[i] += s * h
                xs = xs.view_as(x)
                rec = {}
                vals.append(float(loss(xs if x is p2d else p2d, xs if x is attr else attr, rec)))
                for k in keys:
                    assert torch.equal(rec[k][stable], r64[k][stable]), f"{k} moved under a {h} step"
            fd.view(-1)[i] = (vals[0] - vals[1]) / (2 * h)
        scale = float(gx.abs().max())
        assert scale > 0
        assert float((fd - gx).abs().max()) <= 1e-6 * scale, (fd, gx)


def one_face(p2d, nz, uv=None):
    """A single face as float64 oracle inputs (depth 0); uv: one (u, v) for all three corners."""
    p2d = torch.tensor([p2d], dtype=torch.float64).view(1, 1, 6)
    p3d = torch.zeros(1, 1, 9, dtype=torch.float64)
    p3d[..., 0::3], p3d[..., 1::3] = p2d[..., 0::2], p2d[..., 1::2]
    uv = (0.5, 0.5) if uv is None else uv
    attr = torch.tensor([uv[0], uv[1], 1.0] * 3, dtype=torch.float64).view(1, 1, 9)
    return p3d, p2d, torch.tensor([[[nz]]], dtype=torch.float64), attr


def records(p3d, p2d, nz, attr, H, W):
    r32, r64 = {}, {}
    o32 = M.rasterize(p3d.float(), p2d.float(), nz.float(), attr.float(), H, W, record=r32)
    o64 = M.rasterize(p3d, p2d, nz, attr, H, W, record=r64)
    return r32, r64, o32[0][..., :2], o64[0][..., :2]


def test_stable_pixels_flags_equal_edge_distances():
    """A back face's incentre is equally far from all three edges (closest points on three different edges)."""
    import math
    r = 0.3
    tri = [r * v for a in (90, 210, 330) for v in (math.cos(math.radians(a)), math.sin(math.radians(a)))]
    r32, r64, _, _ = records(*one_face(tri, -1.0), 9, 9)            # pixel (4, 4) has its centre at (0, 0)
    assert int(r64["imidx"].max()) == 0 and int(r64["soft_n"][0, 4, 4]) == 1
    assert float(r64["edge_gap"][0, 4, 4]) < M.EDGE_TIE_REL
    stable = M.stable_pixels(r32, r64)
    assert not bool(stable[0, 4, 4]) and int(stable.sum()) > 40


@pytest.mark.parametrize("filtering,frac", [("bilinear", 1e-7), ("bicubic", 1e-7), ("nearest", 0.5 + 1e-7)])
def test_stable_pixels_flags_texel_fraction(filtering, frac):
    """A covered pixel sampling its texture 1e-7 texel from a floor (or a nearest rounding) boundary."""
    Th, Tw = 8, 12
    k = 5
    if filtering == "bilinear":
        u, v = (k + frac) / (Tw - 1), 1 - (3 + 0.5) / (Th - 1)
    else:                                      # ix = u * Tw - 0.5, iy = (1 - v) * Th - 0.5
        u, v = (k + frac + 0.5) / Tw, 1 - (3.25 + 0.5) / Th
    face = [-0.9, -0.9, 0.9, -0.9, 0.0, 0.9]
    r32, r64, uv32, uv64 = records(*one_face(face, 1.0, (u, v)), 9, 9)
    assert int(r64["imidx"][0, 4, 4]) == 1
    stable = M.stable_pixels(r32, r64, uv32, uv64, (Th, Tw), filtering)
    assert not bool(stable[0, 4, 4])
    # the same face sampling mid-texel is stable
    if filtering == "nearest":
        u = (k + 0.25 + 0.5) / Tw
    else:
        u = (k + 0.5) / (Tw - 1) if filtering == "bilinear" else (k + 0.5 + 0.5) / Tw
    r32, r64, uv32, uv64 = records(*one_face(face, 1.0, (u, v)), 9, 9)
    assert bool(M.stable_pixels(r32, r64, uv32, uv64, (Th, Tw), filtering)[0, 4, 4])


def test_stable_pixels_flags_expanded_box_edge():
    """A face whose expanded bounding box starts exactly at a pixel centre: xmin - expand = x0 = 0."""
    e = M.EXPAND
    r32, r64, _, _ = records(*one_face([e, -0.1, e + 0.3, -0.05, e + 0.1, 0.2], 1.0), 9, 9)
    assert int(r64["imidx"][0, 4, 4]) == 0 and float(r64["box_gap"][0, 4, 4]) < M.BOX_MARGIN
    stable = M.stable_pixels(r32, r64)
    assert not bool(stable[0, 4, 4])
    # one pixel further out the decision is a full pitch away
    assert bool(stable[0, 4, 3])


@pytest.mark.parametrize("H,W", [(17, 33), (40, 56), (64, 96), (250, 90)])
def test_bin_faces_matches_oracle_tiles(sphere, H, W):
    """bin_faces (the kernel's per-tile lists, fp32) holds every face the oracle tests against a pixel of the tile, in
    face order.  Where the expanded box (>= 2 expand wide) spans a pixel pitch the two sets are equal; otherwise the
    tile's list may also hold faces whose box falls between two pixel centres."""
    p3d, p2d, nz, attr = posed(sphere, 2, 4)
    rec = {}
    M.rasterize(p3d, p2d, nz, attr, H, W, record=rec)
    pos = M.bin_faces(p2d, H, W)
    assert tuple(pos.shape) == (2, (H + 15) // 16, (W + 15) // 16, p2d.shape[1])
    exact = 2 * M.EXPAND >= 2 / min(H, W)
    for b in range(2):
        for ty in range(pos.shape[1]):
            for tx in range(pos.shape[2]):
                p = pos[b, ty, tx]
                listed = p[p >= 0]
                assert torch.equal(listed, torch.arange(len(listed)))       # compact positions
                faces = (p >= 0).nonzero()[:, 0].tolist()                    # in face order by construction
                tested = rec["tiles"].get((b, ty, tx), [])
                if exact:
                    assert faces == tested, (b, ty, tx)
                else:
                    assert set(tested) <= set(faces), (b, ty, tx)
    assert int(pos.max()) > 0
