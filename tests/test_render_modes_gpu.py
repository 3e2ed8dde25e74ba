"""Texture filters of Renderer and kaolin's full linear_rasterizer surface on the CUDA rasteriser.

  * bilinear through the filtered entry points = the Renderer entry points (same launch code, kaolin's defaults);
  * linear_rasterizer (any d, points2d / normalz as given, expand / knum / multiplier / delta) against
    oracle/mesh.py:rasterize: face-index buffer exact, fp32 tolerances written at each assert;
  * Renderer(filtering='nearest' | 'bicubic') against torch's grid_sample composition (rendering/fragment_shader.py) and
    against the reference's Renderer (tests/golden/filtering_reference.npz);
  * every new path captured in a CUDA graph replays to its eager result.
The 16-ring procedural sphere and random poses, as in test_mesh_gpu.py."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import mesh as M

sys.path.insert(0, GOLDEN)
import filtering_common as FC        # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def tpl():
    from rendering.mesh_template import MeshTemplate
    path = M.write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16)
    return MeshTemplate(path, device=DEV), M.TemplateData(M.load_obj(path), path)


def scene(T, B, seed, tex_res=32):
    g = torch.Generator().manual_seed(seed)
    mesh_map = torch.randn(B, 3, 32, 32, generator=g) * 0.05
    q = torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=-1)
    s = 0.5 + 0.3 * torch.rand(B, 1, generator=g)
    t = (torch.rand(B, 3, generator=g) - 0.5) * 0.3
    tex = torch.rand(B, 3, tex_res, tex_res, generator=g) * 2 - 1
    vtx = M.transform_vertices(M.get_vertex_positions(T, mesh_map), s, t, q)
    return vtx, tex, g


def rel(a, b):
    return float((a.detach().cpu() - b.detach().cpu()).abs().max()) / max(float(b.detach().abs().max()), 1e-30)


# ---- bilinear: the filtered entry points at the defaults are the Renderer's --------------------------------------------
def test_bilinear_filtered_entry_equals_render_entry(tpl):
    import b3d
    from b3d import lib, ptr, stream_ptr
    from b3d.mesh import face_setup
    from rendering.renderer import Renderer
    mt, T = tpl
    B, H = 2, 64
    vtx, tex, g = scene(T, B, 3)
    uvs, padded = M.adjust_uv_and_texture(T, tex)
    fgeo, fuv, _ = face_setup(vtx.to(DEV), T.faces.to(DEV), uvs.to(DEV), T.face_textures.to(DEV))
    tx = padded.to(DEV).contiguous()
    bg = torch.rand(B, H, H, 3, generator=g).to(DEV)
    F_, Th, Tw = fgeo.shape[1], tx.shape[2], tx.shape[3]
    d_out, d_prob = torch.rand(B, H, H, 3, generator=g).to(DEV), torch.rand(B, H, H, generator=g).to(DEV)
    for bgi in (None, bg):
        outs = []
        for filtered in (False, True):
            o = (torch.empty(B, H, H, dtype=torch.int32, device=DEV), torch.empty(B, H, H, 3, device=DEV),
                 torch.empty(B, H, H, 3, device=DEV), torch.empty(B, H, H, device=DEV))
            gr = (torch.empty(B, F_, 6, device=DEV), torch.empty(B, F_, 6, device=DEV), torch.empty_like(tx))
            if filtered:
                b3d.check(lib.b3d_mesh_render_filtered_fwd(ptr(fgeo), ptr(fuv), ptr(tx), ptr(bgi), B, F_, H, H, Th, Tw, 0,
                                                           *map(ptr, o), stream_ptr()))
                b3d.check(lib.b3d_mesh_render_filtered_bwd(ptr(fgeo), ptr(fuv), ptr(tx), int(bgi is not None), B, F_, H,
                                                           H, Th, Tw, 0, ptr(o[0]), ptr(o[1]), ptr(d_out), ptr(d_prob),
                                                           *map(ptr, gr), stream_ptr()))
            else:
                b3d.check(lib.b3d_mesh_render_fwd(ptr(fgeo), ptr(fuv), ptr(tx), ptr(bgi), B, F_, H, H, Th, Tw,
                                                  *map(ptr, o), stream_ptr()))
                b3d.check(lib.b3d_mesh_render_bwd(ptr(fgeo), ptr(fuv), ptr(tx), int(bgi is not None), B, F_, H, H, Th,
                                                  Tw, ptr(o[0]), ptr(o[1]), ptr(d_out), ptr(d_prob), *map(ptr, gr),
                                                  stream_ptr()))
            outs.append((o, gr))
        (o0, g0), (o1, g1) = outs
        for a, b in zip(o0, o1):
            assert torch.equal(a, b)                          # forward: bit for bit
        for a, b in zip(g0, g1):
            # same kernel, same arguments; only the order of the float atomics may differ between two launches
            assert rel(a, b) < 1e-6
    # Renderer('bilinear') = the entry points above (through face_setup + the index scatter)
    r = Renderer(H, H)
    img, alpha = mt.forward_renderer(r, vtx.to(DEV), tex.to(DEV))
    assert torch.equal(r.last_face_index, o0[0]) and torch.equal(alpha[..., 0], o0[3])


# ---- linear_rasterizer: kaolin's contract -------------------------------------------------------------------------
def kaolin_inputs(T, vtx, g, d):
    p3d, p2d, normal = M.ortho_projection(vtx, T.faces)
    attr = torch.rand(vtx.shape[0], p2d.shape[1], 3 * d, generator=g) * 2 - 1
    return p3d, p2d, normal[:, :, 2:3].contiguous(), attr


def compare_rasterizer(p3d, p2d, nz, attr, H, W, g, check_grads=True, **kw):
    """CUDA raster_attr against oracle rasterize (forward, face-index buffer, gradients); returns the CUDA imfeat."""
    from b3d.mesh import raster_attr
    okw = dict(expand=kw.get("expand", M.EXPAND), knum=kw.get("knum", M.KNUM), mult=kw.get("multiplier", M.MULTIPLIER),
               delta=kw.get("delta", M.DELTA))
    d = attr.shape[2] // 3
    wf, wp = torch.rand(p2d.shape[0], H, W, d, generator=g), torch.rand(p2d.shape[0], H, W, 1, generator=g)
    po, ao = p2d.clone().requires_grad_(True), attr.clone().requires_grad_(True)
    f_o, pr_o, idx_o, _ = FC.rasterize(p3d, po, nz, ao, H, W, **okw)
    gpo, gao = torch.autograd.grad((f_o * wf).sum() + (pr_o * wp).sum(), [po, ao])
    c3, c2, cn, ca = (t.to(DEV).requires_grad_(True) for t in (p3d, p2d, nz, attr))
    f_c, pr_c, idx_c, _ = raster_attr(c3, c2, cn, ca, H, W, **kw)
    assert f_c.shape == (p2d.shape[0], H, W, d) and pr_c.shape == (p2d.shape[0], H, W, 1)
    nbad = int((idx_c.cpu() != idx_o).sum())
    assert nbad == 0, f"face-index buffer differs in {nbad} of {idx_o.numel()} pixels"
    assert float((f_c.detach().cpu() - f_o.detach()).abs().max()) < 2e-5 * float(attr.abs().max())
    assert float((pr_c.detach().cpu() - pr_o.detach()).abs().max()) < 2e-5
    if check_grads:
        g3, g2, gn, ga = torch.autograd.grad((f_c * wf.to(DEV)).sum() + (pr_c * wp.to(DEV)).sum(), [c3, c2, cn, ca])
        assert float(g3.abs().max()) == 0 and float(gn.abs().max()) == 0       # kaolin: no gradient to depth / normalz
        assert rel(g2, gpo) < 2e-3, rel(g2, gpo)
        assert rel(ga, gao) < 2e-3, rel(ga, gao)
    return f_c.detach().cpu(), idx_o


@pytest.mark.parametrize("H", [64, 256])
@pytest.mark.parametrize("d", [1, 3, 4, 16])
def test_linear_rasterizer_attributes(tpl, H, d):
    from rendering.renderer import linear_rasterizer
    _, T = tpl
    vtx, _, g = scene(T, 2, 10 + d)
    p3d, p2d, nz, attr = kaolin_inputs(T, vtx, g, d)
    f_c, idx = compare_rasterizer(p3d, p2d, nz, attr, H, H, g, check_grads=(H == 64))
    assert 0.05 < float((idx > 0).float().mean()) < 0.9
    if d == 3:          # a non-constant third channel is interpolated, not replaced by the hard mask
        assert float((f_c[..., 2][idx > 0] - 1).abs().max()) > 0.1
    # the kaolin-signature wrapper: (width, height, ...) -> the same imfeat
    imfeat, improb = linear_rasterizer(H, H, p3d.to(DEV), p2d.to(DEV), nz.to(DEV), attr.to(DEV))
    assert torch.equal(imfeat.cpu(), f_c)


def test_linear_rasterizer_uses_points2d_and_normalz_as_given(tpl):
    _, T = tpl
    vtx, _, g = scene(T, 2, 21)
    p3d, p2d, nz, attr = kaolin_inputs(T, vtx, g, 3)
    f_ortho, idx_ortho = compare_rasterizer(p3d, p2d, nz, attr, 64, 64, g, check_grads=False)
    # perspective projection: xy / (z0 - z), a points2d that is not points3d's xy
    z = p3d[:, :, 2::3]
    persp = (p2d.view(2, -1, 3, 2) * (2.0 / (2.5 - z)).unsqueeze(-1)).reshape(p2d.shape).contiguous()
    f_p, idx_p = compare_rasterizer(p3d, persp, nz, attr, 64, 64, g)
    assert int((idx_p != idx_ortho).sum()) > 50
    # flipped normals: the back faces become the front faces
    f_n, idx_n = compare_rasterizer(p3d, p2d, -nz, attr, 64, 64, g)
    assert int((idx_n != idx_ortho).sum()) > 50


@pytest.mark.parametrize("kw,H,W", [
    (dict(expand=0.0), 64, 64), (dict(expand=0.05), 64, 64),
    (dict(knum=1), 64, 64), (dict(knum=64), 64, 64),
    (dict(multiplier=500.0), 64, 64), (dict(multiplier=2000.0), 64, 64),
    (dict(delta=1000.0), 64, 64), (dict(delta=20000.0), 64, 64),
    (dict(), 48, 80), (dict(), 80, 48),
])
def test_linear_rasterizer_parameters(tpl, kw, H, W):
    _, T = tpl
    vtx, _, g = scene(T, 2, 30)
    p3d, p2d, nz, attr = kaolin_inputs(T, vtx, g, 3)
    compare_rasterizer(p3d, p2d, nz, attr, H, W, g, **kw)


# ---- texture filters ------------------------------------------------------------------------------------------------
def filter_scene(T, seed, uv_map):
    vtx, tex, g = scene(T, 2, seed, tex_res=16)
    uvs, padded = M.adjust_uv_and_texture(T, tex)
    return vtx, (uvs * uv_map[0] + uv_map[1]).contiguous(), padded.contiguous(), g


@pytest.mark.parametrize("filtering", ["nearest", "bicubic"])
@pytest.mark.parametrize("with_bg", [False, True])
@pytest.mark.parametrize("uv_map", [(1.0, 0.0), (1.3, -0.15)])
def test_renderer_filter_against_grid_sample(tpl, filtering, with_bg, uv_map):
    from b3d.mesh import render
    from rendering.fragment_shader import fragmentshader
    from rendering.renderer import Renderer
    _, T = tpl
    B, H = 2, 64
    vtx, uvs, tex, g = filter_scene(T, 40 + int(with_bg), uv_map)
    bg = torch.rand(B, H, H, 3, generator=g) if with_bg else None
    faces, ft = T.faces.to(DEV), T.face_textures.to(DEV)
    # the same scene unshaded: the kernel's own (u, v, hard mask) per pixel
    uvm, _, idx_u, _ = render(vtx.to(DEV), faces, uvs.to(DEV), None, ft=ft, H=H, W=H)
    uvm = uvm.cpu()
    vc, uc, tc = (t.to(DEV).requires_grad_(True) for t in (vtx, uvs, tex))
    r = Renderer(H, H, filtering=filtering)
    img, alpha, _ = r([vc, faces], uc, tc, ft_fx3=ft, background_image=None if bg is None else bg.to(DEV))
    assert torch.equal(r.last_face_index, idx_u)
    tt = tex.clone().requires_grad_(True)
    ref = fragmentshader(uvm[..., :2], tt, uvm[..., 2:3], filtering=filtering, background_image=bg)
    tol = 1e-6 if filtering == "nearest" else 1e-5
    assert float((img.detach().cpu() - ref.detach()).abs().max()) < tol * float(tex.abs().max())
    _, hard, _ = r([vc.detach(), faces], uc.detach(), tc.detach(), ft_fx3=ft, return_hardmask=True)
    assert torch.equal(hard[..., 0], (idx_u > 0).float())
    # texture gradient against grid_sample's adjoint on the same sampling points
    wi, wa = torch.rand(B, H, H, 3, generator=g), torch.rand(B, H, H, 1, generator=g)
    gt_ref, = torch.autograd.grad((ref * wi).sum(), [tt])
    gv, gu, gt = torch.autograd.grad((img * wi.to(DEV)).sum(), [vc, uc, tc], retain_graph=True)
    assert rel(gt, gt_ref) < 1e-4, rel(gt, gt_ref)
    if filtering == "nearest":
        assert float(gv.abs().max()) == 0 and float(gu.abs().max()) == 0     # grid_sample nearest: no coordinate gradient
    # vertices / uvs (colour and soft-silhouette paths) against torch autograd of the oracle composition
    vo, uo, to = (t.clone().requires_grad_(True) for t in (vtx, uvs, tex))
    img_o, alpha_o, _, _ = FC.render(vo, T.faces, uo, to, T.face_textures, H, H, background_image=bg, filtering=filtering)
    gvo, guo = torch.autograd.grad((img_o * wi).sum() + (alpha_o * wa).sum(), [vo, uo])
    gv, gu = torch.autograd.grad((img * wi.to(DEV)).sum() + (alpha * wa.to(DEV)).sum(), [vc, uc])
    assert rel(gv, gvo) < 2e-3, rel(gv, gvo)
    if filtering == "bicubic":
        assert rel(gu, guo) < 2e-3, rel(gu, guo)
    else:
        assert float(gu.abs().max()) == 0 and float(guo.abs().max()) == 0


def test_renderer_filter_errors():
    from rendering.renderer import Renderer
    for f in ("bilinear", "nearest", "bicubic"):
        assert Renderer(8, 8, filtering=f).filtering == f
    with pytest.raises(ValueError):
        Renderer(8, 8, filtering="area")


def test_filtering_golden(tpl):
    """The CUDA Renderer on the golden's scenes against the reference's Renderer (filtering_reference.npz)."""
    from rendering.renderer import Renderer
    _, T = tpl
    z = np.load(os.path.join(GOLDEN, "filtering_reference.npz"))
    H = int(z["H"][0])
    faces, ft = T.faces.to(DEV), T.face_textures.to(DEV)
    boundary_total = 0
    for si in range(2):
        vtx, uvs, tex, bg = (torch.from_numpy(z[f"s{si}_{k}"]) for k in ("vtx", "uvs", "tex", "bg"))
        # the golden's per-pixel texture coordinates (the oracle rasteriser's) -> pixels near a nearest-rounding boundary
        p3d, p2d, nrm = M.ortho_projection(vtx, T.faces)
        feat, _, idx_o, _ = M.rasterize(p3d, p2d, nrm[:, :, 2:3], FC.uv_attributes(uvs, T.face_textures), H, H)
        Th, Tw = tex.shape[2], tex.shape[3]
        ix = (feat[..., 0] * 2 - 1 + 1) * (Tw / 2) - 0.5
        iy = (-(feat[..., 1] * 2 - 1) + 1) * (Th / 2) - 0.5
        near = (((ix - ix.floor() - 0.5).abs() < 1e-4) | ((iy - iy.floor() - 0.5).abs() < 1e-4)) & (idx_o > 0)
        for f in ("nearest", "bicubic"):
            r = Renderer(H, H, filtering=f)
            img, alpha, _ = r([vtx.to(DEV), faces], uvs.to(DEV), tex.to(DEV), ft_fx3=ft)
            img_bg, hard, _ = r([vtx.to(DEV), faces], uvs.to(DEV), tex.to(DEV), ft_fx3=ft, background_image=bg.to(DEV),
                                return_hardmask=True)
            assert torch.equal(r.last_face_index.cpu(), idx_o)
            assert float((alpha.cpu() - torch.from_numpy(z[f"s{si}_{f}_alpha"])).abs().max()) < 2e-5
            assert torch.equal(hard.cpu() > 0.5, torch.from_numpy(z[f"s{si}_{f}_hard"]) > 0.5)
            for got, key in ((img, "img"), (img_bg, "img_bg")):
                err = (got.cpu() - torch.from_numpy(z[f"s{si}_{f}_{key}"])).abs().amax(-1)
                if f == "nearest":
                    assert float(err[~near].max()) < 2e-5
                    boundary_total += int(near.sum())
                else:
                    assert float(err.max()) < 2e-5
    print(f"nearest: {boundary_total} pixel renders within 1e-4 texel of a rounding boundary (excluded)")


# ---- CUDA graphs ------------------------------------------------------------------------------------------------------
def graph_equals_eager(step, leaves):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            for t in leaves:
                t.grad = None
            eager = [o.detach().clone() for o in step()]
            eager_grads = [t.grad.clone() for t in leaves]
    torch.cuda.current_stream().wait_stream(side)
    for t in leaves:
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(list(outs) + [t.grad for t in leaves], eager + eager_grads):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6 * float(b.abs().max()))


@pytest.mark.parametrize("filtering", ["nearest", "bicubic"])
def test_filtered_render_in_cuda_graph(tpl, filtering):
    from rendering.renderer import Renderer
    _, T = tpl
    vtx, uvs, tex, g = filter_scene(T, 50, (1.0, 0.0))
    vc, uc, tc = (t.to(DEV).requires_grad_(True) for t in (vtx, uvs, tex))
    faces, ft = T.faces.to(DEV), T.face_textures.to(DEV)
    r = Renderer(64, 64, filtering=filtering)
    w = torch.rand(2, 64, 64, 3, generator=g).to(DEV)

    def step():
        img, alpha, _ = r([vc, faces], uc, tc, ft_fx3=ft)
        ((img * w).sum() + alpha.sum()).backward()
        return img, alpha

    graph_equals_eager(step, [vc, uc, tc])


@pytest.mark.parametrize("d,kw", [(3, dict()), (16, dict(expand=0.05, knum=8, multiplier=2000.0, delta=20000.0))])
def test_linear_rasterizer_in_cuda_graph(tpl, d, kw):
    from rendering.renderer import linear_rasterizer
    _, T = tpl
    vtx, _, g = scene(T, 2, 60)
    p3d, p2d, nz, attr = kaolin_inputs(T, vtx, g, d)
    c3, cn = p3d.to(DEV), nz.to(DEV)
    c2, ca = p2d.to(DEV).requires_grad_(True), attr.to(DEV).requires_grad_(True)
    w = torch.rand(2, 64, 64, d, generator=g).to(DEV)

    def step():
        imfeat, improb = linear_rasterizer(64, 64, c3, c2, cn, ca, **kw)
        ((imfeat * w).sum() + improb.sum()).backward()
        return imfeat, improb

    graph_equals_eager(step, [c2, ca])
