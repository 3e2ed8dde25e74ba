"""Oracle side of the texture-filter and kaolin-parameter tests (tests/test_render_modes_*.py).

`render` is oracle/mesh.py:render with the reference's filter switch: the same ortho_projection -> rasterize -> (u, v, 1)
attribute split, shaded by rendering/fragment_shader.py:fragmentshader, whose non-bilinear modes go to F.grid_sample with
its defaults exactly as the reference's fragment_shader.py:11-17 does.  tests/golden/filtering_reference.npz (the
reference's Renderer run unmodified) pins it.

`multiplier` lets oracle/mesh.py:rasterize run with a non-default kaolin multiplier: the function reads its pixel
centres and face windows from the module constant MULTIPLIER, so the constant is set for the duration of the call.
"""
import contextlib

import torch

from oracle import mesh as M


@contextlib.contextmanager
def multiplier(m):
    saved = M.MULTIPLIER
    M.MULTIPLIER = float(m)
    try:
        yield
    finally:
        M.MULTIPLIER = saved


def rasterize(p3d, p2d, normalz, attr, H, W, expand=M.EXPAND, knum=M.KNUM, mult=M.MULTIPLIER, delta=M.DELTA):
    """oracle/mesh.py:rasterize with any kaolin multiplier."""
    with multiplier(mult):
        return M.rasterize(p3d, p2d, normalz, attr, H, W, expand=expand, knum=knum, multiplier=float(mult), delta=delta)


def uv_attributes(uv, ft):
    """Renderer.forward's (u, v, 1) per face corner, renderer.py:54-58."""
    c = [uv[:, ft[:, i], :] for i in range(3)]
    one = torch.ones_like(c[0][:, :, :1])
    return torch.cat((c[0], one, c[1], one, c[2], one), dim=2)


def render(points, faces, uv, texture, ft=None, H=256, W=256, background_image=None, return_hardmask=False,
           filtering="bilinear"):
    """Renderer(H, W, filtering).forward -> (imrender, improb | hardmask, normal1, imidx)."""
    from rendering.fragment_shader import fragmentshader
    ft = faces if ft is None else ft
    p3d, p2d, normal = M.ortho_projection(points, faces)
    imfeat, improb, imidx, _ = M.rasterize(p3d, p2d, normal[:, :, 2:3], uv_attributes(uv, ft), H, W)
    hard = imfeat[..., 2:3]
    img = fragmentshader(imfeat[..., :2], texture, hard, filtering=filtering, background_image=background_image)
    return img, (hard if return_hardmask else improb), M.datanormalize(normal, 2), imidx
