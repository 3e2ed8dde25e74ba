"""The CUDA mesh rasteriser and its adjoint against the fp64 oracle, with the discrete decisions pinned.

oracle/mesh.py:rasterize runs twice, in fp32 and in fp64, recording every discrete decision per pixel; stable_pixels
keeps the pixels where both runs take the same decisions with a margin (coverage and depth winner, expanded-box
membership, the knum cap, the closest edge, the segment clamp, the texel floor / round, the p_k clamp).  Per case:
  1. the face-index buffer equals the fp32 oracle's on every pixel;
  2. unstable pixels get zero upstream gradients on all three sides; their forward values are held to the fp32 oracle
     at the bound of test_mesh_gpu.py (2e-5);
  3. at most 1 % of the pixels are unstable, and every behaviour a case targets keeps stable pixels;
  4. forward on stable pixels and every gradient, max-norm: |cuda - o64| <= 4 |o32 - o64| + 1e-5 max|o64|;
  5. per face: |g_cuda[f] - g64[f]| <= 4 |g32[f] - g64[f]| + 1e-5 |g64[f]| + 1e-7 max_f |g64[f]|, so that small faces
     do not hide behind the largest one.
Gradients are those to the vertices (through face_setup), uvs or attributes and texture; the Python render path returns
none for the background.  Each case prints its unstable-pixel fraction, its worst err / tol ratio and how many faces past
the shared-memory accumulator capacity of a tile list it checked."""
import math
import os
import sys
import tempfile

import pytest
import torch

from conftest import GOLDEN
from oracle import mesh as M

sys.path.insert(0, GOLDEN)
import filtering_common as FC        # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CAPN = 768                 # per-tile shared-memory accumulators of the backward: 768 faces x 12 slots
FILT = {"bilinear": 0, "nearest": 1, "bicubic": 2}


def capn_attr(d):
    return CAPN * 12 // (6 + 3 * d)


# ---- inputs ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tpl():
    tmp = tempfile.mkdtemp()
    out = {}
    for rings in (16, 31):
        path = M.write_uvsphere_obj(os.path.join(tmp, f"uvsphere_{rings}rings.obj"), rings=rings)
        out[rings] = M.TemplateData(M.load_obj(path), path)
    return out


def posed(T, B, seed, scale=(0.5, 0.8), shift=0.3, tex_hw=(32, 32)):
    """Seeded random deformation and pose of a template, with a random texture -> (vtx, uvs [B,T,2], padded texture)."""
    g = torch.Generator().manual_seed(seed)
    mesh_map = torch.randn(B, 3, 32, 32, generator=g) * 0.05
    q = torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=-1)
    s = scale[0] + (scale[1] - scale[0]) * torch.rand(B, 1, generator=g)
    t = (torch.rand(B, 3, generator=g) - 0.5) * shift
    vtx = M.transform_vertices(M.get_vertex_positions(T, mesh_map), s, t, q)
    uvs, tex = M.adjust_uv_and_texture(T, torch.rand(B, 3, *tex_hw, generator=g) * 2 - 1)
    return vtx, uvs.contiguous(), tex.contiguous()


def small_sphere(T, radius, tilt):
    """The undeformed template scaled to `radius`, tilted about x by `tilt` radians, centred on the image centre."""
    c, s = math.cos(tilt), math.sin(tilt)
    R = torch.tensor([[1.0, 0, 0], [0, c, -s], [0, s, c]])
    return (T.vertices @ R.T * radius).unsqueeze(0)


def weights(B, H, W, C, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, H, W, C, generator=g) * 2 - 1, torch.rand(B, H, W, 1, generator=g) * 2 - 1


# ---- the comparison rule --------------------------------------------------------------------------------------------
class Rule:
    def __init__(self, name):
        self.name, self.worst = name, 0.0

    def maxnorm(self, what, cuda, o32, o64, where=None):
        c, a, b = (t.detach().cpu().double() for t in (cuda, o32, o64))
        if where is not None:
            c, a, b = c[where], a[where], b[where]
        tol = 4 * float((a - b).abs().max()) + 1e-5 * float(b.abs().max())
        err = float((c - b).abs().max())
        self.worst = max(self.worst, err / tol if tol > 0 else (math.inf if err > 0 else 0.0))
        assert err <= tol, f"{self.name} {what}: |cuda - o64| = {err:.3e} > {tol:.3e}"

    def per_face(self, what, cuda, o32, o64):
        """cuda / o32 / o64 [B,F,K] per-face gradients -> the per-face norms of o64 (for the callers' own asserts)."""
        c, a, b = (t.detach().cpu().double() for t in (cuda, o32, o64))
        n64 = b.norm(dim=-1)
        tol = 4 * (a - b).norm(dim=-1) + 1e-5 * n64 + 1e-7 * float(n64.max())
        err = (c - b).norm(dim=-1)
        ratio = torch.where(tol > 0, err / tol.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
        self.worst = max(self.worst, float(ratio.max()))
        bad = (err > tol).nonzero().tolist()
        assert not bad, (f"{self.name} {what}: {len(bad)} faces outside the per-face rule, e.g. (b, f) = {bad[:5]}, "
                         f"err {[float(err[tuple(i)]) for i in bad[:5]]} tol {[float(tol[tuple(i)]) for i in bad[:5]]}")
        return n64


def oracle_raster(p3d, p2d, nz, attr, H, W, dt, params):
    """fp32 or fp64 oracle forward with decisions recorded; p2d / attr are returned as the autograd leaves."""
    p2 = p2d.detach().to(dt).requires_grad_(True)
    at = attr.detach().to(dt).requires_grad_(True)
    rec = {}
    kw = dict(expand=params.get("expand", M.EXPAND), knum=params.get("knum", M.KNUM), delta=params.get("delta", M.DELTA))
    mult = params.get("multiplier", M.MULTIPLIER)
    with FC.multiplier(mult):
        feat, prob, idx, _ = M.rasterize(p3d.to(dt), p2, nz.to(dt), at, H, W, multiplier=float(mult), record=rec, **kw)
    return dict(feat=feat, prob=prob, idx=idx, p2d=p2, attr=at, rec=rec)


def uv_cols(g):
    """[B,F,9] gradient of the (u, v, 1) corner attributes -> [B,F,6] of the corner uvs (the kernel's fuv layout)."""
    return g[..., [0, 1, 3, 4, 6, 7]]


def scatter(per_face, index, n):
    """[B,F,3,2] per-corner values summed onto [B,n,2] by index [F,3] (the adjoint of a gather)."""
    B = per_face.shape[0]
    out = per_face.new_zeros(B, n, 2)
    for i in range(3):
        out.index_add_(1, index[:, i], per_face[:, :, i])
    return out


def budget(rule, stable, targets=()):
    frac = 1 - float(stable.float().mean())
    assert frac <= 0.01, f"{rule.name}: {frac:.2%} of the pixels are unstable"
    for what, m in targets:
        assert int((m & stable).sum()) > 0, f"{rule.name}: no stable pixel left for {what}"
    return frac


def report(rule, frac, n_overflow=0):
    print(f"\n[{rule.name}] unstable {frac:.3%}, worst err/tol {rule.worst:.3f}, overflow-position faces {n_overflow}")


# ---- render (UV and shaded modes) -----------------------------------------------------------------------------------
def cuda_faces(verts, faces, uv, ft, tex, bg, H, W, filt, w_out, w_prob):
    """The render entry points called directly: -> imidx, imout, improb, per-face dfp2d [B,F,6], dfuv [B,F,6], dtex."""
    import b3d
    from b3d import lib, ptr, stream_ptr
    from b3d.mesh import face_setup
    fgeo, fuv, _ = face_setup(verts, faces, uv, ft)
    B, F = fgeo.shape[0], fgeo.shape[1]
    imidx = torch.empty(B, H, W, dtype=torch.int32, device=DEV)
    imwei, imout = torch.empty(B, H, W, 3, device=DEV), torch.empty(B, H, W, 3, device=DEV)
    improb = torch.empty(B, H, W, device=DEV)
    dfp2d, dfuv = torch.empty(B, F, 6, device=DEV), torch.empty(B, F, 6, device=DEV)
    o = (imidx, imwei, imout, improb)
    if tex is None:
        b3d.check(lib.b3d_mesh_render_fwd(ptr(fgeo), ptr(fuv), None, None, B, F, H, W, 0, 0, *map(ptr, o), stream_ptr()))
        b3d.check(lib.b3d_mesh_render_bwd(ptr(fgeo), ptr(fuv), None, 0, B, F, H, W, 0, 0, ptr(imidx), ptr(imwei),
                                          ptr(w_out), ptr(w_prob), ptr(dfp2d), ptr(dfuv), None, stream_ptr()))
        dtex = None
    else:
        Th, Tw = tex.shape[2], tex.shape[3]
        dtex = torch.empty_like(tex)
        b3d.check(lib.b3d_mesh_render_filtered_fwd(ptr(fgeo), ptr(fuv), ptr(tex), ptr(bg), B, F, H, W, Th, Tw, filt,
                                                   *map(ptr, o), stream_ptr()))
        b3d.check(lib.b3d_mesh_render_filtered_bwd(ptr(fgeo), ptr(fuv), ptr(tex), int(bg is not None), B, F, H, W, Th,
                                                   Tw, filt, ptr(imidx), ptr(imwei), ptr(w_out), ptr(w_prob),
                                                   ptr(dfp2d), ptr(dfuv), ptr(dtex), stream_ptr()))
    return imidx, imout, improb.unsqueeze(-1), dfp2d, dfuv, dtex


def shade(orc, tex, bg, filtering, dt):
    """The oracle run's shaded image (fragment_shader.py) or, without a texture, its (u, v, hard mask)."""
    from rendering.fragment_shader import fragmentshader
    if tex is None:
        return orc["feat"][..., :3], None
    t = tex.detach().to(dt).requires_grad_(True)
    b = None if bg is None else bg.to(dt)
    return fragmentshader(orc["feat"][..., :2], t, orc["feat"][..., 2:3], filtering=filtering, background_image=b), t


def check_render(name, vtx, faces, uv, ft, tex, H, W, filtering="bilinear", bg=None, seed=0, orcs=None, targets=(),
                 overflow=False):
    """One render case: the CUDA render (public path and entry points) against the fp32 / fp64 oracle."""
    from b3d.mesh import render
    rule = Rule(name)
    B, F, P = vtx.shape[0], faces.shape[0], vtx.shape[1]
    p3d, p2d, normal = M.ortho_projection(vtx, faces)
    nz = normal[:, :, 2:3]
    if orcs is None:
        attr = FC.uv_attributes(uv, ft)
        orcs = {dt: oracle_raster(p3d, p2d, nz, attr, H, W, dt, {}) for dt in (torch.float32, torch.float64)}
    o32, o64 = orcs[torch.float32], orcs[torch.float64]
    hw = None if tex is None else (tex.shape[2], tex.shape[3])
    stable = M.stable_pixels(o32["rec"], o64["rec"], o32["feat"][..., :2], o64["feat"][..., :2], hw, filtering) \
        if tex is not None else M.stable_pixels(o32["rec"], o64["rec"])
    frac = budget(rule, stable, targets)
    w_out, w_prob = weights(B, H, W, 3, seed)
    keep = stable.unsqueeze(-1).to(w_out.dtype)
    w_out, w_prob = w_out * keep, w_prob * keep

    img, leaves, grads = {}, {}, {}
    for dt, orc in orcs.items():
        im, t = shade(orc, tex, bg, filtering, dt)
        img[dt] = im
        lv = [orc["p2d"], orc["attr"]] + ([t] if t is not None else [])
        loss = (im * w_out.to(dt)).sum() + (orc["prob"] * w_prob.to(dt)).sum()
        g = list(torch.autograd.grad(loss, lv, retain_graph=True))
        g[1] = g[1].view(B, F, 3, -1)[..., :3].reshape(B, F, 9)      # the (u, v, 1) corner attributes
        grads[dt] = g

    vc = vtx.to(DEV).requires_grad_(True)
    uc = uv.to(DEV).requires_grad_(True)
    tc = None if tex is None else tex.to(DEV).requires_grad_(True)
    bgc = None if bg is None else bg.to(DEV)
    out, prob, idx, _ = render(vc, faces.to(DEV), uc, tc, ft=ft.to(DEV), background=bgc, H=H, W=W, filtering=filtering)
    leaves_c = [vc, uc] + ([tc] if tc is not None else [])
    gc = torch.autograd.grad((out * w_out.to(DEV)).sum() + (prob * w_prob.to(DEV)).sum(), leaves_c)
    idx2, out2, prob2, dfp2d, dfuv, dtex = cuda_faces(vc.detach(), faces.to(DEV), uc.detach(), ft.to(DEV),
                                                      None if tc is None else tc.detach(), bgc, H, W, FILT[filtering],
                                                      w_out.to(DEV).contiguous(), w_prob[..., 0].to(DEV).contiguous())
    assert torch.equal(idx, idx2) and torch.equal(out, out2) and torch.equal(prob, prob2)

    # 1. face-index buffer, bit for bit
    nbad = int((idx.cpu() != o32["idx"]).sum())
    assert nbad == 0, f"{name}: face-index buffer differs from the fp32 oracle in {nbad} pixels"
    # 2. unstable pixels: forward at the fp32 bound
    un = ~stable
    if bool(un.any()):
        for c, o in ((out, img[torch.float32]), (prob, o32["prob"])):
            e = float((c.detach().cpu()[un] - o.detach()[un]).abs().max())
            assert e < 2e-5 * max(1.0, float(o.detach().abs().max())), f"{name}: unstable-pixel forward off by {e}"
    # 4. forward on stable pixels, gradients max-norm
    rule.maxnorm("image", out, img[torch.float32], img[torch.float64], stable)
    rule.maxnorm("improb", prob, o32["prob"], o64["prob"], stable)
    fl = faces.long()
    gv = {dt: scatter(g[0].view(B, F, 3, 2), fl, P) for dt, g in grads.items()}
    assert float(gc[0][..., 2].abs().max()) == 0
    rule.maxnorm("d vertices", gc[0][..., :2], gv[torch.float32], gv[torch.float64])
    tl = ft.long()
    gu = {dt: scatter(uv_cols(g[1]).view(B, F, 3, 2), tl, uv.shape[1]) for dt, g in grads.items()}
    rule.maxnorm("d uv", gc[1], gu[torch.float32], gu[torch.float64])
    if tex is not None:
        rule.maxnorm("d texture", gc[2], grads[torch.float32][2], grads[torch.float64][2])
        rule.maxnorm("d texture (entry)", dtex, grads[torch.float32][2], grads[torch.float64][2])
    # 5. per face
    n_p = rule.per_face("d p2d", dfp2d, grads[torch.float32][0], grads[torch.float64][0])
    n_u = rule.per_face("d fuv", dfuv, uv_cols(grads[torch.float32][1]), uv_cols(grads[torch.float64][1]))
    n_over = 0
    if overflow:
        pos = M.bin_faces(p2d, H, W)
        assert int(pos.max()) >= CAPN, f"{name}: no tile list reaches {CAPN} faces"
        over = (pos >= CAPN).flatten(1, 2).any(1)             # [B,F] faces listed past the capacity of some tile
        live = over & ((n_p > 0) | (n_u > 0))
        n_over = int(live.sum())
        assert n_over >= 10, f"{name}: only {n_over} overflow-position faces carry an fp64 gradient"
    report(rule, frac, n_over)
    return dict(stable=stable, o32=o32, o64=o64, dfp2d=dfp2d, dfuv=dfuv, idx=idx.cpu(), grads=grads)


# ---- linear_rasterizer (attributes) ---------------------------------------------------------------------------------
def check_attr(name, p3d, p2d, nz, attr, H, W, params=None, seed=0, orcs=None, col=None, targets=(), overflow=False):
    """raster_attr against the oracle; orcs / col: oracle runs over wider attributes, of which [col, col + d) per
    corner are these."""
    from b3d.mesh import raster_attr
    params = params or {}
    rule = Rule(name)
    B, F, d = p2d.shape[0], p2d.shape[1], attr.shape[2] // 3
    if orcs is None:
        orcs = {dt: oracle_raster(p3d, p2d, nz, attr, H, W, dt, params) for dt in (torch.float32, torch.float64)}
    col = col or 0
    o32, o64 = orcs[torch.float32], orcs[torch.float64]
    stable = M.stable_pixels(o32["rec"], o64["rec"])
    frac = budget(rule, stable, targets)
    w_out, w_prob = weights(B, H, W, d, seed)
    keep = stable.unsqueeze(-1).to(w_out.dtype)
    w_out, w_prob = w_out * keep, w_prob * keep
    feat, grads = {}, {}
    for dt, orc in orcs.items():
        dw = orc["attr"].shape[2] // 3
        feat[dt] = orc["feat"][..., col:col + d]
        loss = (feat[dt] * w_out.to(dt)).sum() + (orc["prob"] * w_prob.to(dt)).sum()
        g2, ga = torch.autograd.grad(loss, [orc["p2d"], orc["attr"]], retain_graph=True)
        grads[dt] = (g2, ga.view(B, F, 3, dw)[..., col:col + d].reshape(B, F, 3 * d))
    c3, c2, cn, ca = (t.to(DEV).requires_grad_(True) for t in (p3d, p2d, nz, attr))
    kw = {k: params[k] for k in ("expand", "knum", "multiplier", "delta") if k in params}
    f_c, pr_c, idx_c, _ = raster_attr(c3, c2, cn, ca, H, W, **kw)
    g2c, gac = torch.autograd.grad((f_c * w_out.to(DEV)).sum() + (pr_c * w_prob.to(DEV)).sum(), [c2, ca])
    nbad = int((idx_c.cpu() != o32["idx"]).sum())
    assert nbad == 0, f"{name}: face-index buffer differs from the fp32 oracle in {nbad} pixels"
    un = ~stable
    if bool(un.any()):
        e = float((f_c.detach().cpu()[un] - feat[torch.float32].detach()[un]).abs().max())
        assert e < 2e-5 * float(attr.abs().max()), f"{name}: unstable-pixel imfeat off by {e}"
        e = float((pr_c.detach().cpu()[un] - o32["prob"].detach()[un]).abs().max())
        assert e < 2e-5, f"{name}: unstable-pixel improb off by {e}"
    rule.maxnorm("imfeat", f_c, feat[torch.float32], feat[torch.float64], stable)
    rule.maxnorm("improb", pr_c, o32["prob"], o64["prob"], stable)
    rule.maxnorm("d points2d", g2c, grads[torch.float32][0], grads[torch.float64][0])
    rule.maxnorm("d attr", gac, grads[torch.float32][1], grads[torch.float64][1])
    n_p = rule.per_face("d points2d", g2c, grads[torch.float32][0], grads[torch.float64][0])
    n_a = rule.per_face("d attr", gac, grads[torch.float32][1], grads[torch.float64][1])
    n_over = 0
    if overflow:
        capn = capn_attr(d)
        pos = M.bin_faces(p2d, H, W, expand=params.get("expand", M.EXPAND),
                          multiplier=params.get("multiplier", M.MULTIPLIER))
        assert int(pos.max()) >= capn, f"{name}: no tile list reaches {capn} faces"
        over = (pos >= capn).flatten(1, 2).any(1)
        n_over = int((over & ((n_p > 0) | (n_a > 0))).sum())
        assert n_over >= 10, f"{name}: only {n_over} overflow-position faces carry an fp64 gradient"
    report(rule, frac, n_over)
    return dict(stable=stable, o32=o32, o64=o64, rec=o32["rec"])


def kaolin_inputs(vtx, faces, d, seed):
    p3d, p2d, normal = M.ortho_projection(vtx, faces)
    g = torch.Generator().manual_seed(seed)
    attr = torch.rand(vtx.shape[0], p2d.shape[1], 3 * d, generator=g) * 2 - 1
    return p3d, p2d, normal[:, :, 2:3].contiguous(), attr


# ---- cases ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(17, 33), (40, 72), (250, 90)])
@pytest.mark.parametrize("with_bg", [False, True])
def test_partial_tiles(tpl, H, W, with_bg):
    T = tpl[16]
    vtx, uvs, tex = posed(T, 3, 200 + H, scale=(1.0, 1.2))          # large enough to reach the partial tiles
    bg = torch.rand(3, H, W, 3, generator=torch.Generator().manual_seed(W)) if with_bg else None
    r = check_render(f"partial tiles {H}x{W} bg={with_bg}", vtx, T.faces, uvs, T.face_textures, tex, H, W, bg=bg,
                     seed=H + W)
    # the last, partial tile row and column hold stable covered pixels and stable soft-silhouette pixels
    cov = r["idx"] > 0
    edge = torch.zeros_like(cov)
    edge[:, (H // 16) * 16:, :] = True
    edge[:, :, (W // 16) * 16:] = True
    assert int((edge & r["stable"] & cov).sum()) > 0
    assert int((edge & r["stable"] & (r["o64"]["rec"]["soft_n"] > 0)).sum()) > 0


def overflow_sphere(T):
    """960-face sphere, undeformed, centred on the middle 16x16 tile of a 48x48 image and small enough that every face's
    expanded box reaches that tile: its list holds all 960 faces.  Tilted so that the last faces in face order (the
    rings around the south pole) face the camera and cover pixels."""
    return small_sphere(T, 0.29, -1.0)


def test_list_overflow_render(tpl):
    T = tpl[16]
    vtx = overflow_sphere(T)
    g = torch.Generator().manual_seed(7)
    uvs, tex = M.adjust_uv_and_texture(T, torch.rand(1, 3, 32, 32, generator=g) * 2 - 1)
    check_render("list overflow render (capn 768)", vtx, T.faces, uvs.contiguous(), T.face_textures, tex.contiguous(),
                 48, 48, seed=8, overflow=True)


@pytest.mark.parametrize("d", [3, 16])
def test_list_overflow_attr(tpl, d):
    T = tpl[16]
    p3d, p2d, nz, attr = kaolin_inputs(overflow_sphere(T), T.faces, d, 9 + d)
    check_attr(f"list overflow raster_attr d={d} (capn {capn_attr(d)})", p3d, p2d, nz, attr, 48, 48, seed=d,
               overflow=True)


@pytest.mark.parametrize("knum", [1, 2, 30, 4096])
def test_knum_cap(tpl, knum):
    T = tpl[31]
    vtx, _, _ = posed(T, 2, 200, scale=(0.25, 0.35), shift=0.1)      # small faces: up to ~40 candidates a pixel
    p3d, p2d, nz, attr = kaolin_inputs(vtx, T.faces, 3, 201)
    H = W = 64
    orcs = {dt: oracle_raster(p3d, p2d, nz, attr, H, W, dt, dict(knum=knum)) for dt in (torch.float32, torch.float64)}
    rec = orcs[torch.float64]["rec"]
    unc = rec["imidx"] == 0
    cut = unc & (rec["cand"] > knum)
    if knum == 4096:
        assert not bool(cut.any()) and torch.equal(rec["soft_n"], rec["cand"])
        targets = (("uncovered pixels with candidates", unc & (rec["cand"] > 0)),)
    else:
        targets = (("pixels with more than knum candidates", cut),)
    check_attr(f"knum {knum}", p3d, p2d, nz, attr, H, W, dict(knum=knum), seed=knum, orcs=orcs, targets=targets)


@pytest.mark.parametrize("rings", [16, 31])
def test_benchmark_shapes(tpl, rings):
    """960 faces (cfg2 / cfg3) and the 1920-face 31-ring template (cfg4) at 256^2, B = 2, every output mode.  One oracle
    rasterisation per precision carries the (u, v, 1) corner attributes and the d = 1, 3, 16 attributes side by side."""
    T = tpl[rings]
    B, H = 2, 256
    vtx, uvs, tex = posed(T, B, 300 + rings)
    p3d, p2d, normal = M.ortho_projection(vtx, T.faces)
    nz = normal[:, :, 2:3].contiguous()
    F = p2d.shape[1]
    g = torch.Generator().manual_seed(rings)
    extra = {d: torch.rand(B, F, 3 * d, generator=g) * 2 - 1 for d in (1, 3, 16)}
    parts = [FC.uv_attributes(uvs, T.face_textures)] + [extra[d] for d in (1, 3, 16)]
    wide = torch.cat([p.view(B, F, 3, -1) for p in parts], dim=3).reshape(B, F, -1)
    orcs = {dt: oracle_raster(p3d, p2d, nz, wide, H, H, dt, {}) for dt in (torch.float32, torch.float64)}
    check_render(f"{F} faces 256^2 uv", vtx, T.faces, uvs, T.face_textures, None, H, H, seed=1, orcs=orcs)
    for i, f in enumerate(("bilinear", "nearest", "bicubic")):
        check_render(f"{F} faces 256^2 {f}", vtx, T.faces, uvs, T.face_textures, tex, H, H, filtering=f, seed=2 + i,
                     orcs=orcs)
    col = 3
    for d in (1, 3, 16):
        check_attr(f"{F} faces 256^2 attr d={d}", p3d, p2d, nz, extra[d], H, H, seed=10 + d, orcs=orcs, col=col)
        col += d


@pytest.mark.parametrize("variant", ["Th!=Tw", "2x2", "uv past [0,1]"])
def test_texture_edges(tpl, variant):
    T = tpl[16]
    tex_hw = {"Th!=Tw": (24, 40), "2x2": (2, 2), "uv past [0,1]": (16, 16)}[variant]
    vtx, uvs, tex = posed(T, 2, 400 + tex_hw[1], tex_hw=tex_hw)
    if variant == "uv past [0,1]":
        uvs = (uvs * 1.3 - 0.15).contiguous()
    H = 64
    orcs = {dt: oracle_raster(*M.ortho_projection(vtx, T.faces)[:2],
                              M.ortho_projection(vtx, T.faces)[2][:, :, 2:3], FC.uv_attributes(uvs, T.face_textures),
                              H, H, dt, {}) for dt in (torch.float32, torch.float64)}
    for i, f in enumerate(("bilinear", "nearest", "bicubic")):
        targets = ()
        if variant == "uv past [0,1]":
            Th, Tw = tex.shape[2], tex.shape[3]
            ix, iy = M.texel_coords(orcs[torch.float64]["feat"][..., :2].detach(), Th, Tw, f)
            # a tap of the filter footprint falls outside the texture, into the zero padding
            reach = 1.0 if f != "bicubic" else 2.0
            out = (ix.floor() < 0) | (ix.floor() + reach > Tw - 1) | (iy.floor() < 0) | (iy.floor() + reach > Th - 1)
            if f == "nearest":
                out = (ix.round() < 0) | (ix.round() > Tw - 1) | (iy.round() < 0) | (iy.round() > Th - 1)
            targets = (("taps in the zero padding", out & (orcs[torch.float64]["rec"]["imidx"] > 0)),)
        check_render(f"texture {variant} {tuple(tex.shape[2:])} {f}", vtx, T.faces, uvs, T.face_textures, tex, H, H,
                     filtering=f, seed=20 + i, orcs=orcs, targets=targets)


def test_flipped_normals(tpl):
    """Negated normalz: the back faces become the front faces (kaolin draws faces with normalz >= 0)."""
    T = tpl[16]
    vtx, _, _ = posed(T, 2, 500)
    p3d, p2d, nz, attr = kaolin_inputs(vtx, T.faces, 3, 501)
    r = check_attr("flipped normals", p3d, p2d, -nz, attr, 64, 64, seed=5)
    won = r["rec"]["imidx"]
    assert bool((won > 0).any())
    b_ix = torch.arange(2).view(2, 1, 1).expand_as(won)[won > 0]
    assert bool((nz[b_ix, (won[won > 0] - 1).long(), 0] <= 0).all())


def test_duplicated_face(tpl):
    """Visible faces appended a second time: equal depth, so face order keeps the first copy; the copy gets no
    colour-path gradient (uvs), and only what its soft silhouette gives to the 2-D vertices."""
    T = tpl[16]
    vtx, uvs, tex = posed(T, 1, 600)
    p3d, p2d, normal = M.ortho_projection(vtx, T.faces)
    front = (normal[0, :, 2] > 0).nonzero()[:, 0]
    dup = front[::7][:40]
    faces = torch.cat([T.faces, T.faces[dup]])
    ft = torch.cat([T.face_textures, T.face_textures[dup]])
    F0 = T.faces.shape[0]
    r = check_render("duplicated faces", vtx, faces, uvs, ft, tex, 64, 64, seed=6)
    assert int((r["idx"] > F0).sum()) == 0                       # no copy ever wins
    covered_dups = torch.isin(r["idx"].long() - 1, dup)
    assert int(covered_dups.sum()) > 0
    assert float(r["dfuv"][0, F0:].abs().max()) == 0
    assert float(r["grads"][torch.float64][1][0, F0:].abs().max()) == 0
    assert float(r["dfuv"][0, dup].abs().max()) > 0


@pytest.mark.parametrize("params", [dict(expand=0.0), dict(multiplier=500.0), dict(multiplier=2000.0),
                                    dict(delta=1000.0), dict(delta=20000.0)])
def test_raster_parameters(tpl, params):
    T = tpl[16]
    vtx, _, _ = posed(T, 2, 700)
    p3d, p2d, nz, attr = kaolin_inputs(vtx, T.faces, 3, 701)
    r = check_attr(f"params {params}", p3d, p2d, nz, attr, 64, 64, params, seed=7)
    soft = (r["rec"]["imidx"] == 0) & (r["rec"]["soft_n"] > 0)
    if params.get("expand", M.EXPAND) > 0:
        assert int((soft & r["stable"]).sum()) > 0
