"""Generate tests/golden/filtering_reference.npz by running the REFERENCE's rendering/renderer.py:Renderer.forward,
unmodified, on the CPU with filtering='nearest' and 'bicubic' (authoring container only):
    python tests/golden/make_golden_filtering.py
The construction is make_golden_renderer.py's: kaolin's `linear_rasterizer` / `datanormalize` are the oracle's
restatements (oracle/mesh.py, parity unpinned).  What this pins is the wiring around the rasteriser for the filters the
reference hands to F.grid_sample (fragment_shader.py:11-17): its defaults align_corners=False and padding_mode='zeros',
the v flip, the hard-mask multiply / background lerp and return_hardmask.  The second scene's uvs are pushed past
[0, 1] so that zero padding is exercised.
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference/code")

from oracle import mesh as M                      # noqa: E402

calls = []


def linear_rasterizer(width, height, points3d_bxfx9, points2d_bxfx6, normalz_bxfx1, vertex_attr_bxfx3d):
    calls.append((width, height))
    imfeat, improb, _, _ = M.rasterize(points3d_bxfx9, points2d_bxfx6, normalz_bxfx1, vertex_attr_bxfx3d, height, width)
    return imfeat, improb


mods = {n: types.ModuleType(n) for n in ("kaolin", "kaolin.graphics", "kaolin.graphics.dib_renderer",
                                         "kaolin.graphics.dib_renderer.rasterizer", "kaolin.graphics.dib_renderer.utils")}
mods["kaolin.graphics.dib_renderer.rasterizer"].linear_rasterizer = linear_rasterizer
mods["kaolin.graphics.dib_renderer.utils"].datanormalize = M.datanormalize
sys.modules.update(mods)

from rendering.renderer import Renderer       # noqa: E402  (reference, unmodified)

FILTERS = ("nearest", "bicubic")
# per scene: uv affine map u' = a * u + b (scene 1 reaches outside [0, 1] -> zero padding)
UV_MAPS = ((1.0, 0.0), (1.3, -0.15))


def main():
    out = {}
    path = M.write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16)
    T = M.TemplateData(M.load_obj(path), path)
    g = torch.Generator().manual_seed(31)
    B, H = 2, 48
    for si, (ua, ub) in enumerate(UV_MAPS):
        mesh_map = torch.randn(B, 3, 32, 32, generator=g) * 0.05
        q = torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=-1)
        s, t = 0.5 + 0.3 * torch.rand(B, 1, generator=g), (torch.rand(B, 3, generator=g) - 0.5) * 0.3
        tex = torch.rand(B, 3, 16, 16, generator=g) * 2 - 1
        bg = torch.rand(B, H, H, 3, generator=g)
        vtx = M.transform_vertices(M.get_vertex_positions(T, mesh_map), s, t, q)
        uvs, padded = M.adjust_uv_and_texture(T, tex)
        uvs = uvs * ua + ub
        out.update({f"s{si}_vtx": vtx.numpy(), f"s{si}_uvs": uvs.numpy(), f"s{si}_tex": padded.numpy(),
                    f"s{si}_bg": bg.numpy()})
        for f in FILTERS:
            r = Renderer(H, H, filtering=f)
            img, alpha, _ = r([vtx, T.faces], uvs, padded, ft_fx3=T.face_textures)
            img_bg, hard, _ = r([vtx, T.faces], uvs, padded, ft_fx3=T.face_textures, background_image=bg,
                                return_hardmask=True)
            out.update({f"s{si}_{f}_img": img.numpy(), f"s{si}_{f}_alpha": alpha.numpy(),
                        f"s{si}_{f}_img_bg": img_bg.numpy(), f"s{si}_{f}_hard": hard.numpy()})
    out["H"] = np.array([H])
    assert all(c == (H, H) for c in calls) and len(calls) == 2 * len(UV_MAPS) * len(FILTERS)
    p = os.path.join(HERE, "filtering_reference.npz")
    np.savez_compressed(p, **out)
    print("wrote", p, os.path.getsize(p), "bytes")


if __name__ == "__main__":
    main()
