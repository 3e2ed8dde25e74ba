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
    """kaolin.graphics.dib_renderer.rasterizer.linear_rasterizer: -> (imfeat [B,H,W,d], improb [B,H,W,1]).

    points2d and normalz are used as given (any projection, any front-face test), vertex_attr carries any number d of
    values per face corner, and expand / knum / multiplier / delta default to kaolin's 0.02 / 30 / 1000 / 7000.
    Differentiable w.r.t. points2d and vertex_attr; points3d (only its depths are read) and normalz get zero gradients,
    as in kaolin."""
    imfeat, improb, _, _ = _m.raster_attr(points3d_bxfx9, points2d_bxfx6, normalz_bxfx1, vertex_attr_bxfx3d, height,
                                          width, expand=expand, knum=knum, multiplier=multiplier, delta=delta)
    return imfeat, improb


class Renderer(nn.Module):
    def __init__(self, height, width, filtering='bilinear'):
        super().__init__()
        _m.filter_id(filtering)           # 'bilinear' | 'nearest' | 'bicubic', else ValueError (as grid_sample)
        self.height, self.width, self.filtering = height, width, filtering

    def forward(self, points, uv_bxpx2, texture_bx3xthxtw, ft_fx3=None, background_image=None,
                return_hardmask=False):
        """points = [vertices B×P×3, faces F×3]; returns (imrender B×H×W×3, improb | hardmask B×H×W×1,
        unit face normals B×F×3) like the reference."""
        verts, faces = points
        imrender, improb, imidx, normal1 = _m.render(verts, faces, uv_bxpx2, texture_bx3xthxtw,
                                                     ft=ft_fx3, background=background_image,
                                                     H=self.height, W=self.width, filtering=self.filtering)
        self.last_face_index = imidx          # face id + 1 per pixel, 0 = background (visibility buffer)
        if return_hardmask:
            improb = (imidx > 0).to(imrender.dtype).unsqueeze(-1)
        return imrender, improb, normal1
