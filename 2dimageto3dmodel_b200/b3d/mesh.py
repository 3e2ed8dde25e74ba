"""Mesh render ops over libb3d: kaolin-free DIB-R rasteriser + fragment shader (autograd wrappers).

Reference call sites: /root/reference/code/rendering/renderer.py:39-77 (Renderer.forward),
renderer.py:60-67 (kaolin linear_rasterizer), fragment_shader.py:22-37.
"""
import torch

from . import B3DError, check, dev, lib, ptr, stream_ptr


_i32_cache = {}


def _i32(t, name):
    """Index tensors arrive as int64 (the reference's LongTensors); the kernels take int32.  The converted
    copy is cached per source tensor (template topology never changes) so no cast kernel runs per step."""
    if t.dtype == torch.int32:
        return dev(t, name, torch.int32)
    key = (t.data_ptr(), tuple(t.shape), t._version, str(t.device))
    hit = _i32_cache.get(key)
    if hit is None or hit[0] is not t:
        # the entry keeps the SOURCE tensor alive: its address cannot be recycled for another index tensor of the same
        # shape while the converted copy is cached (a different tensor at the same key simply replaces the entry)
        if len(_i32_cache) > 64:
            _i32_cache.clear()
        hit = _i32_cache[key] = (t, dev(t.to(torch.int32), name, torch.int32))
    return hit[1]


def face_setup(verts, faces, uv=None, ft=None, want_normals=True):
    """verts [B,P,3], faces [F,3], uv [B,T,2]|[T,2], ft [F,3] -> fgeo [B,F,12], fuv [B,F,6], normal1 [B,F,3]."""
    verts = dev(verts, "vertices")
    faces = _i32(faces, "faces")
    B, P, _ = verts.shape
    F = faces.shape[0]
    fgeo = torch.empty(B, F, 12, device=verts.device, dtype=torch.float32)
    normal1 = torch.empty(B, F, 3, device=verts.device, dtype=torch.float32) if want_normals else None
    fuv, T, batched = None, 0, 0
    if uv is not None:
        ft = _i32(faces if ft is None else ft, "face_textures")
        batched = 1 if uv.dim() == 3 else 0
        if batched and uv.stride(0) == 0:       # .expand()-ed template uvs (mesh_template.py:161)
            uv, batched = uv[0], 0
        uv = dev(uv, "uv")
        T = uv.shape[-2]
        fuv = torch.empty(B, F, 6, device=verts.device, dtype=torch.float32)
    check(lib.b3d_mesh_face_setup(ptr(verts), ptr(faces), ptr(uv), batched, ptr(ft), B, P, F, T, ptr(fgeo), ptr(fuv),
                                  ptr(normal1), stream_ptr(verts)))
    return fgeo, fuv, normal1


# Renderer(filtering=...) -> B3D_FILTER_* of include/b3d.h (grid_sample's modes the shader kernels are built for)
FILTERS = {"bilinear": 0, "nearest": 1, "bicubic": 2}


class _Render(torch.autograd.Function):
    """(vertices, uv, texture) -> (imout [B,H,W,3], improb [B,H,W,1], imidx [B,H,W] int32, normal1 [B,F,3]).
    filt: B3D_FILTER_* id of the texture filter (ignored without a texture)."""

    @staticmethod
    def forward(ctx, verts, uv, texture, faces, ft, background, H, W, filt=0):
        verts_d = dev(verts.detach(), "vertices")
        uv_d = uv.detach()
        fgeo, fuv, normal1 = face_setup(verts_d, faces, uv_d, ft)
        B, F = fgeo.shape[0], fgeo.shape[1]
        tex = dev(texture.detach(), "texture") if texture is not None else None
        Th, Tw = (tex.shape[2], tex.shape[3]) if tex is not None else (0, 0)
        if tex is not None and (tex.dim() != 4 or tex.shape[1] != 3 or tex.shape[0] != B):
            # the shader kernels are built for RGB textures (every reference call site passes 3 channels)
            raise B3DError(f"render: texture must be [B={B},3,Th,Tw], got {tuple(tex.shape)}")
        bg = dev(background.detach(), "background_image") if background is not None else None
        if bg is not None and tuple(bg.shape) != (B, H, W, 3):
            raise B3DError(f"render: background_image must be [B={B},{H},{W},3], got {tuple(bg.shape)}")
        d = verts_d.device
        imidx = torch.empty(B, H, W, device=d, dtype=torch.int32)
        imwei = torch.empty(B, H, W, 3, device=d, dtype=torch.float32)
        imout = torch.empty(B, H, W, 3, device=d, dtype=torch.float32)
        improb = torch.empty(B, H, W, 1, device=d, dtype=torch.float32)
        if tex is not None:
            check(lib.b3d_mesh_render_filtered_fwd(ptr(fgeo), ptr(fuv), ptr(tex), ptr(bg), B, F, H, W, Th, Tw, filt,
                                                   ptr(imidx), ptr(imwei), ptr(imout), ptr(improb), stream_ptr(verts_d)))
        else:
            check(lib.b3d_mesh_render_fwd(ptr(fgeo), ptr(fuv), None, None, B, F, H, W, 0, 0, ptr(imidx), ptr(imwei),
                                          ptr(imout), ptr(improb), stream_ptr(verts_d)))
        ctx.save_for_backward(fgeo, fuv, tex if tex is not None else torch.empty(0), imidx, imwei,
                              _i32(faces, "faces"), _i32(faces if ft is None else ft, "face_textures"))
        ctx.cfg = (H, W, Th, Tw, tex is not None, bg is not None, verts.shape, uv.shape, uv.dim() == 3 and uv.stride(0) != 0)
        ctx.filt = filt
        ctx.mark_non_differentiable(imidx, normal1)
        return imout, improb, imidx, normal1

    @staticmethod
    def backward(ctx, d_imout, d_improb, _d_idx, _d_n):
        fgeo, fuv, tex, imidx, imwei, faces, ft = ctx.saved_tensors
        H, W, Th, Tw, has_tex, has_bg, vshape, uvshape, uv_batched = ctx.cfg
        B, F = fgeo.shape[0], fgeo.shape[1]
        d = fgeo.device
        d_imout = dev(d_imout, "grad imrender") if d_imout is not None else torch.zeros(B, H, W, 3, device=d)
        d_improb = dev(d_improb, "grad improb") if d_improb is not None else None
        dfp2d = torch.empty(B, F, 6, device=d, dtype=torch.float32)
        dfuv = torch.empty(B, F, 6, device=d, dtype=torch.float32)
        dtex = torch.empty(B, 3, Th, Tw, device=d, dtype=torch.float32) if has_tex else None
        if has_tex:
            check(lib.b3d_mesh_render_filtered_bwd(ptr(fgeo), ptr(fuv), ptr(tex), int(has_bg), B, F, H, W, Th, Tw,
                                                   ctx.filt, ptr(imidx), ptr(imwei), ptr(d_imout), ptr(d_improb),
                                                   ptr(dfp2d), ptr(dfuv), ptr(dtex), stream_ptr(fgeo)))
        else:
            check(lib.b3d_mesh_render_bwd(ptr(fgeo), ptr(fuv), None, int(has_bg), B, F, H, W, Th, Tw, ptr(imidx),
                                          ptr(imwei), ptr(d_imout), ptr(d_improb), ptr(dfp2d), ptr(dfuv), None,
                                          stream_ptr(fgeo)))
        # scatter the per-face-corner gradients back to vertices / uvs (482 vertices: plumbing)
        dverts = torch.zeros(vshape, device=d, dtype=torch.float32)
        fl = faces.long()
        g = dfp2d.view(B, F, 3, 2)
        for i in range(3):
            dverts[:, :, :2].index_add_(1, fl[:, i], g[:, :, i])
        duv = None
        if ctx.needs_input_grad[1]:
            tl = ft.long()
            gu = dfuv.view(B, F, 3, 2)
            T = uvshape[-2]
            duv_b = torch.zeros(B, T, 2, device=d, dtype=torch.float32)
            for i in range(3):
                duv_b.index_add_(1, tl[:, i], gu[:, :, i])
            duv = duv_b if len(uvshape) == 3 and uv_batched else (duv_b.sum(0) if len(uvshape) == 2 else duv_b)
        return dverts, duv, dtex, None, None, None, None, None, None


def filter_id(filtering):
    """grid_sample mode name -> B3D_FILTER_* id; ValueError for a mode the shader is not built for (as grid_sample)."""
    try:
        return FILTERS[filtering]
    except (KeyError, TypeError):
        raise ValueError(f"texture filtering must be one of {sorted(FILTERS)}, got {filtering!r}") from None


def render(verts, faces, uv, texture, ft=None, background=None, H=256, W=256, filtering="bilinear"):
    if verts.dim() != 3 or verts.size(-1) != 3:
        raise B3DError(f"vertices must be [B,P,3], got {tuple(verts.shape)}")
    return _Render.apply(verts, uv, texture, faces, ft, background, int(H), int(W), filter_id(filtering))


# kaolin linear_rasterizer's keyword defaults (expand, knum, multiplier, delta)
RASTER_DEFAULTS = (0.02, 30, 1000.0, 7000.0)


def raster_params(expand=None, knum=None, multiplier=None, delta=None):
    """kaolin's keyword arguments with its defaults filled in, checked as the C entry points check them."""
    e, k, m, dl = (d if v is None else v for v, d in zip((expand, knum, multiplier, delta), RASTER_DEFAULTS))
    if int(k) != k or k < 1:
        raise B3DError(f"linear_rasterizer: knum={k}, need an integer >= 1")
    if not m > 0 or not dl > 0 or not e >= 0:
        raise B3DError(f"linear_rasterizer: need multiplier > 0, delta > 0, expand >= 0 (got {m}, {dl}, {e})")
    return float(e), int(k), float(m), float(dl)


class _RasterAttr(torch.autograd.Function):
    """kaolin linear_rasterizer on its own inputs: (points3d [B,F,9], points2d [B,F,6], normalz [B,F,1], attr [B,F,3d])
    -> (imfeat [B,H,W,d], improb [B,H,W,1], imidx [B,H,W] int32, imwei [B,H,W,3]).  Differentiable w.r.t. points2d and
    attr; points3d / normalz get zero gradients (kaolin semantics)."""

    @staticmethod
    def forward(ctx, p3d, p2d, normalz, attr, H, W, params):
        expand, knum, mult, delta = params
        p3d_d = dev(p3d.detach(), "points3d")
        p2d_d = dev(p2d.detach(), "points2d")
        nz = dev(normalz.detach(), "normalz")
        at = dev(attr.detach(), "vertex_attr")
        B, F = p2d_d.shape[0], p2d_d.shape[1]
        d = at.shape[2] // 3
        dv = p2d_d.device
        fgeo = torch.empty(B, F, 12, device=dv, dtype=torch.float32)
        imidx = torch.empty(B, H, W, device=dv, dtype=torch.int32)
        imwei = torch.empty(B, H, W, 3, device=dv, dtype=torch.float32)
        imfeat = torch.empty(B, H, W, d, device=dv, dtype=torch.float32)
        improb = torch.empty(B, H, W, 1, device=dv, dtype=torch.float32)
        st = stream_ptr(p2d_d)
        check(lib.b3d_mesh_face_pack(ptr(p3d_d), ptr(p2d_d), ptr(nz), mult, B, F, ptr(fgeo), st))
        check(lib.b3d_mesh_raster_attr_fwd(ptr(fgeo), ptr(at), d, B, F, H, W, expand, knum, mult, delta, ptr(imidx),
                                           ptr(imwei), ptr(imfeat), ptr(improb), st))
        ctx.save_for_backward(fgeo, at, imidx, imwei)
        ctx.cfg = (H, W, params, p3d.shape, normalz.shape)
        ctx.mark_non_differentiable(imidx, imwei)
        return imfeat, improb, imidx, imwei

    @staticmethod
    def backward(ctx, d_imfeat, d_improb, _d_idx, _d_wei):
        fgeo, at, imidx, imwei = ctx.saved_tensors
        H, W, (expand, knum, mult, delta), s3, sn = ctx.cfg
        B, F, d = fgeo.shape[0], fgeo.shape[1], at.shape[2] // 3
        dv = fgeo.device
        d_imfeat = dev(d_imfeat, "grad imfeat") if d_imfeat is not None else torch.zeros(B, H, W, d, device=dv)
        d_improb = dev(d_improb, "grad improb") if d_improb is not None else None
        dp2d = torch.empty(B, F, 6, device=dv, dtype=torch.float32)
        dattr = torch.empty(B, F, 3 * d, device=dv, dtype=torch.float32)
        check(lib.b3d_mesh_raster_attr_bwd(ptr(fgeo), ptr(at), d, B, F, H, W, expand, knum, mult, delta, ptr(imidx),
                                           ptr(imwei), ptr(d_imfeat), ptr(d_improb), ptr(dp2d), ptr(dattr),
                                           stream_ptr(fgeo)))
        d3 = torch.zeros(s3, device=dv) if ctx.needs_input_grad[0] else None
        dn = torch.zeros(sn, device=dv) if ctx.needs_input_grad[2] else None
        return d3, dp2d, dn, dattr, None, None, None


def raster_attr(points3d, points2d, normalz, vertex_attr, H, W, expand=None, knum=None, multiplier=None, delta=None):
    """kaolin linear_rasterizer(W, H, points3d, points2d, normalz, vertex_attr, expand, knum, multiplier, delta) with
    the face-index and barycentric buffers: -> (imfeat [B,H,W,d], improb [B,H,W,1], imidx [B,H,W] int32 face + 1,
    imwei [B,H,W,3])."""
    params = raster_params(expand, knum, multiplier, delta)
    if points2d.dim() != 3 or points2d.shape[2] != 6:
        raise B3DError(f"linear_rasterizer: points2d must be [B,F,6], got {tuple(points2d.shape)}")
    B, F = points2d.shape[0], points2d.shape[1]
    if tuple(points3d.shape) != (B, F, 9):
        raise B3DError(f"linear_rasterizer: points3d must be [{B},{F},9], got {tuple(points3d.shape)}")
    if tuple(normalz.shape) != (B, F, 1):
        raise B3DError(f"linear_rasterizer: normalz must be [{B},{F},1], got {tuple(normalz.shape)}")
    if vertex_attr.dim() != 3 or tuple(vertex_attr.shape[:2]) != (B, F) or vertex_attr.shape[2] < 3 \
            or vertex_attr.shape[2] % 3:
        raise B3DError(f"linear_rasterizer: vertex_attr must be [{B},{F},3d] with d >= 1, got {tuple(vertex_attr.shape)}")
    if int(H) < 1 or int(W) < 1:
        raise B3DError(f"linear_rasterizer: bad image size {H} x {W}")
    return _RasterAttr.apply(points3d, points2d, normalz, vertex_attr, int(H), int(W), params)


@torch.no_grad()
def render_indices(verts, faces, uv, ft, H, W, out=None):
    """Unshaded forward render (no texture): -> (imidx [B,H,W] int32, imwei [B,H,W,3], fuv [B,F,6]), the inputs of
    `texel_visibility`.  out: optional (imidx, imwei, imout, improb) buffers of at least B samples, reused across calls
    (imout [B,H,W,3] and improb [B,H,W,1] are written but not returned)."""
    fgeo, fuv, _ = face_setup(verts, faces, uv, ft, want_normals=False)
    B, F = fgeo.shape[0], fgeo.shape[1]
    d = fgeo.device
    if out is None:
        out = (torch.empty(B, H, W, device=d, dtype=torch.int32), torch.empty(B, H, W, 3, device=d),
               torch.empty(B, H, W, 3, device=d), torch.empty(B, H, W, 1, device=d))
    shapes = ((H, W), (H, W, 3), (H, W, 3), (H, W, 1))
    dtypes = (torch.int32, torch.float32, torch.float32, torch.float32)
    for t, s, dt in zip(out, shapes, dtypes):
        if not (t.is_cuda and t.dtype == dt and t.is_contiguous() and t.shape[0] >= B and tuple(t.shape[1:]) == s):
            raise B3DError(f"render_indices: buffer {tuple(t.shape)} {t.dtype} cannot hold [{B},{','.join(map(str, s))}] {dt}")
    imidx, imwei, imout, improb = (t[:B] for t in out)
    check(lib.b3d_mesh_render_fwd(ptr(fgeo), ptr(fuv), None, None, B, F, H, W, 0, 0, ptr(imidx), ptr(imwei), ptr(imout),
                                  ptr(improb), stream_ptr(fgeo)))
    return imidx, imwei, fuv


def texel_visibility(imidx, imwei, fuv, Th, Tw, symmetric, out=None, words=None):
    """Texels of the texture behind a forward render whose gradient d(render)/d(texture) with an all-ones upstream gradient
    is > 0, computed from the render's index buffers (no adjoint, no float atomics).  Th x Tw: the padded texture the shader
    samples (MeshTemplate.adjust_uv_and_texture); symmetric: circpad(., 1) seam (Tw - 2 columns out), else the appended
    column 0 (Tw - 1 columns out).  -> uint8 [B, Th, Tw_out] of 0 / 1.  out / words: optional reusable buffers of at least B
    samples (words: int32 [B, ceil(Th * Tw_out / 32)])."""
    imidx = dev(imidx, "imidx", torch.int32)
    imwei = dev(imwei, "imwei")
    fuv = dev(fuv, "fuv")
    B, H, W = imidx.shape
    F = fuv.shape[1]
    Tw_out = Tw - (2 if symmetric else 1)
    if tuple(imwei.shape) != (B, H, W, 3) or fuv.dim() != 3 or tuple(fuv.shape) != (B, F, 6):
        raise B3DError(f"texel_visibility: imidx {tuple(imidx.shape)}, imwei {tuple(imwei.shape)}, fuv {tuple(fuv.shape)}")
    if Th < 2 or Tw_out < (2 if symmetric else 1):
        raise B3DError(f"texel_visibility: bad padded texture size {Th} x {Tw}")
    nwords = (Th * Tw_out + 31) // 32
    if out is None:
        out = torch.empty(B, Th, Tw_out, device=imidx.device, dtype=torch.uint8)
    if words is None:
        words = torch.empty(B, nwords, device=imidx.device, dtype=torch.int32)
    if not (out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and out.shape[0] >= B
            and tuple(out.shape[1:]) == (Th, Tw_out)):
        raise B3DError(f"texel_visibility: out must be a contiguous uint8 CUDA tensor [>={B},{Th},{Tw_out}]")
    if not (words.is_cuda and words.dtype == torch.int32 and words.is_contiguous() and words.shape[0] >= B
            and tuple(words.shape[1:]) == (nwords,)):
        raise B3DError(f"texel_visibility: words must be a contiguous int32 CUDA tensor [>={B},{nwords}]")
    out = out[:B]
    check(lib.b3d_texel_visibility(ptr(imidx), ptr(imwei), ptr(fuv), B, F, H, W, int(Th), int(Tw), int(bool(symmetric)),
                                   ptr(words), ptr(out), stream_ptr(imidx)))
    return out


class _FaceNormals(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces):
        v = dev(verts.detach(), "vertices")
        fi = _i32(faces, "faces")
        if v.dim() != 3 or v.shape[2] != 3 or fi.dim() != 2 or fi.shape[1] != 3:
            raise B3DError(f"face_normals: vertices {tuple(v.shape)} / faces {tuple(fi.shape)}")
        B, V, _ = v.shape
        out = torch.empty(B, fi.shape[0], 3, device=v.device, dtype=torch.float32)
        check(lib.b3d_face_normals_fwd(ptr(v), ptr(fi), B, V, fi.shape[0], ptr(out), stream_ptr(v)))
        ctx.save_for_backward(v, fi)
        return out

    @staticmethod
    def backward(ctx, g):
        v, fi = ctx.saved_tensors
        B, V, _ = v.shape
        g = dev(g, "grad")
        dv = torch.empty_like(v)
        check(lib.b3d_face_normals_bwd(ptr(v), ptr(fi), ptr(g), B, V, fi.shape[0], ptr(dv), stream_ptr(v)))
        return dv, None


def face_normals(verts, faces):
    """Unit face normals [B,F,3] of vertices [B,V,3] (MeshTemplate.compute_normals, rendering/mesh_template.py:113-123)."""
    return _FaceNormals.apply(verts, faces)


class _FlatLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, norms, ff):
        n = dev(norms.detach(), "norms")
        ffi = _i32(ff, "ff")
        B, F, _ = n.shape
        loss = torch.empty(1, device=n.device, dtype=torch.float32)
        check(lib.b3d_flat_loss_fwd(ptr(n), ptr(ffi), B, F, ffi.shape[1], ptr(loss), stream_ptr(n)))
        ctx.save_for_backward(n, ffi)
        return loss.view(())

    @staticmethod
    def backward(ctx, g):
        n, ffi = ctx.saved_tensors
        B, F, _ = n.shape
        g = dev(g.reshape(1), "grad")
        dn = torch.empty_like(n)
        check(lib.b3d_flat_loss_bwd(ptr(n), ptr(ffi), B, F, ffi.shape[1], ptr(g), ptr(dn), stream_ptr(n)))
        return dn, None


def flat_loss(norms, ff):
    """loss_flat of utils/losses.py:5-17 on face normals [B,F,3] with adjacency ff [F,K]."""
    return _FlatLoss.apply(norms, ff)


# criterion -> (forward + IoU counts, backward) entry points of csrc/loss_kernels.cu
_RGBA_LOSS = {"mse": ("b3d_rgba_mse_iou_fwd", "b3d_rgba_mse_bwd"), "l1": ("b3d_rgba_l1_iou_fwd", "b3d_rgba_l1_bwd")}


class _RgbaLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, alpha, target, criterion):
        fwd, bwd = _RGBA_LOSS[criterion]
        im = dev(image.detach(), "image_pred")
        al = dev(alpha.detach(), "alpha_pred")
        tg = dev(target.detach(), "X_real")
        B, H, W, _ = im.shape
        if tg.shape != (B, 4, H, W) or al.numel() != B * H * W:
            raise B3DError(f"rgba_{criterion}_iou: shapes image {tuple(im.shape)} alpha {tuple(al.shape)} "
                           f"target {tuple(tg.shape)}")
        loss = torch.empty(1, device=im.device, dtype=torch.float32)
        counts = torch.empty(B, 2, device=im.device, dtype=torch.int32)
        check(getattr(lib, fwd)(ptr(im), ptr(al), ptr(tg), B, H, W, ptr(loss), ptr(counts), stream_ptr(im)))
        ctx.save_for_backward(im, al, tg)
        ctx.ashape, ctx.bwd = alpha.shape, bwd
        ctx.mark_non_differentiable(counts)
        return loss.view(()), counts

    @staticmethod
    def backward(ctx, g, _gc):
        im, al, tg = ctx.saved_tensors
        B, H, W, _ = im.shape
        g = dev(g.reshape(1), "grad")
        di, da = torch.empty_like(im), torch.empty_like(al)
        check(getattr(lib, ctx.bwd)(ptr(im), ptr(al), ptr(tg), B, H, W, ptr(g), ptr(di), ptr(da), stream_ptr(im)))
        return di, da.view(ctx.ashape), None, None


def _rgba_loss_iou(image_pred, alpha_pred, X_real, criterion):
    loss, counts = _RgbaLoss.apply(image_pred, alpha_pred, X_real, criterion)
    c = counts.to(torch.float32)
    return loss, (c[:, 0] / c[:, 1]).mean()


def rgba_mse_iou(image_pred, alpha_pred, X_real):
    """Fused form of run_reconstruction.py:429-436:
        X_fake = cat(image_pred, alpha_pred, 3).permute(0,3,1,2); nn.MSELoss()(X_fake, X_real); mean_iou(...)
    -> (recon_loss, miou); miou carries no gradient, like the reference's torch.no_grad() block."""
    return _rgba_loss_iou(image_pred, alpha_pred, X_real, "mse")


def rgba_l1_iou(image_pred, alpha_pred, X_real):
    """rgba_mse_iou with the reference's --loss l1 criterion nn.L1Loss() (run_reconstruction.py:347-352): the mean of
    |X_fake - X_real|; its gradient is torch's sign(d) / n, 0 where prediction and target are equal."""
    return _rgba_loss_iou(image_pred, alpha_pred, X_real, "l1")
