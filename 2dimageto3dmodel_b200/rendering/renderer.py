"""Drop-in for /root/reference/code/rendering/renderer.py — with the kaolin dependency replaced.

`Renderer.forward` (reference :39-77) = ortho_projection (:9-28) -> kaolin DIB-R `linear_rasterizer`
(:60-67) -> `fragmentshader` (:72).  Here those three stages are two sm_90a kernels of libb3d
(csrc/mesh_kernels.cu: per-face setup, then a tile-binned rasteriser with the shader fused in).
`linear_rasterizer` / `datanormalize` below stand in for the two kaolin functions the reference imports.
"""
import torch
import torch.nn as nn

from b3d import mesh as _m


def ortho_projection(points_bxpx3, faces_fx3):
    """(points3d [B,F,9], points2d [B,F,6], normal [B,F,3]) as renderer.py:9-28 returns them."""
    idx = faces_fx3.long()
    tri = [points_bxpx3[:, idx[:, k], :] for k in range(3)]
    normal = torch.cross(tri[1] - tri[0], tri[2] - tri[0], dim=2)
    return torch.cat(tri, dim=2), torch.cat([t[:, :, :2] for t in tri], dim=2), normal


def datanormalize(x, axis):
    """kaolin.graphics.dib_renderer.utils.datanormalize."""
    return x / (x.norm(dim=axis, keepdim=True) + 1e-8)


def linear_rasterizer(width, height, points3d_bxfx9, points2d_bxfx6, normalz_bxfx1, vertex_attr_bxfx3d,
                      expand=None, knum=None, multiplier=None, delta=None):
    """Signature of kaolin.graphics.dib_renderer.rasterizer.linear_rasterizer; only the defaults the
    reference uses (expand .02, knum 30, multiplier 1000, delta 7000) and d=3 attributes (u,v,1) are built."""
    for v, dflt in ((expand, 0.02), (knum, 30), (multiplier, 1000), (delta, 7000)):
        if v is not None and v != dflt:
            raise _m.B3DError("linear_rasterizer: only kaolin's default expand/knum/multiplier/delta are supported")
    B, F, _ = points3d_bxfx9.shape
    # re-pack as an indexed mesh with 3F private vertices so the same kernels apply
    verts = points3d_bxfx9.reshape(B, 3 * F, 3)
    faces = torch.arange(3 * F, device=verts.device, dtype=torch.int32).view(F, 3)
    if vertex_attr_bxfx3d.shape[2] != 9:
        raise _m.B3DError("linear_rasterizer: expected 3 attributes per vertex (u, v, 1)")
    uv = vertex_attr_bxfx3d.reshape(B, 3 * F, 3)[:, :, :2].contiguous()
    imfeat, improb, _, _ = _m.render(verts, faces, uv, None, ft=faces, H=height, W=width)
    return imfeat, improb


class Renderer(nn.Module):
    def __init__(self, height, width, filtering='bilinear'):
        super().__init__()
        if filtering != 'bilinear':
            raise _m.B3DError("Renderer: only bilinear texture filtering is built (the reference default)")
        self.height, self.width, self.filtering = height, width, filtering

    def forward(self, points, uv_bxpx2, texture_bx3xthxtw, ft_fx3=None, background_image=None,
                return_hardmask=False):
        """points = [vertices B×P×3, faces F×3]; returns (imrender B×H×W×3, improb | hardmask B×H×W×1,
        unit face normals B×F×3) like the reference."""
        verts, faces = points
        imrender, improb, imidx, normal1 = _m.render(verts, faces, uv_bxpx2, texture_bx3xthxtw,
                                                     ft=ft_fx3, background=background_image,
                                                     H=self.height, W=self.width)
        self.last_face_index = imidx          # face id + 1 per pixel, 0 = background (visibility buffer)
        if return_hardmask:
            improb = (imidx > 0).to(imrender.dtype).unsqueeze(-1)
        return imrender, improb, normal1
