"""Timing of the mesh rasteriser's modes on one GPU at cfg2's mesh size: B 16, 256^2 renders of the 960-face 16-ring
procedural sphere, a 128 x 130 (seam-padded) texture, random poses.  Each case is one forward + backward through the
public Python entry points (autograd included):
  bilinear / nearest / bicubic   b3d.mesh.render (Renderer's path) with that texture filter;
  attr d=3 / d=16                b3d.mesh.raster_attr (linear_rasterizer) at kaolin's defaults;
  attr d=3 / d=16 params         expand 0.05, knum 64, multiplier 2000, delta 20000.
CUDA events around windows of --iters calls, the cases alternated window by window over --rounds rounds after a
warm-up; the median per call and the min-max over the rounds.  Prints the card's name and power limit and one JSON
line.  CUDA only."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "2dimageto3dmodel_b200"))
sys.path.insert(0, ROOT)

import numpy as np   # noqa: E402
import torch         # noqa: E402

DEV = "cuda:0"
B, RES, TEX = 16, 256, 128
NONDEFAULT = dict(expand=0.05, knum=64, multiplier=2000.0, delta=20000.0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def inputs():
    from oracle import mesh as M
    path = M.write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16)
    T = M.TemplateData(M.load_obj(path), path)
    g = torch.Generator().manual_seed(0)
    mesh_map = torch.randn(B, 3, 32, 32, generator=g) * 0.05
    q = torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=-1)
    s, t = 0.5 + 0.3 * torch.rand(B, 1, generator=g), (torch.rand(B, 3, generator=g) - 0.5) * 0.3
    vtx = M.transform_vertices(M.get_vertex_positions(T, mesh_map), s, t, q)
    uvs, tex = M.adjust_uv_and_texture(T, torch.rand(B, 3, TEX, TEX, generator=g) * 2 - 1)
    p3d, p2d, normal = M.ortho_projection(vtx, T.faces)
    return T, vtx, uvs.contiguous(), tex.contiguous(), p3d, p2d, normal[:, :, 2:3].contiguous(), g


def cases():
    from b3d.mesh import raster_attr, render
    T, vtx, uvs, tex, p3d, p2d, nz, g = inputs()
    faces, ft = T.faces.to(DEV), T.face_textures.to(DEV)
    vc, uc, tc = (x.to(DEV).requires_grad_(True) for x in (vtx, uvs, tex))
    wi, wa = torch.rand(B, RES, RES, 3, generator=g).to(DEV), torch.rand(B, RES, RES, 1, generator=g).to(DEV)
    out = {}
    for f in ("bilinear", "nearest", "bicubic"):
        def run(f=f):
            img, alpha, _, _ = render(vc, faces, uc, tc, ft=ft, H=RES, W=RES, filtering=f)
            torch.autograd.grad((img * wi).sum() + (alpha * wa).sum(), [vc, uc, tc])
        out[f] = run
    c3, cn, c2 = p3d.to(DEV), nz.to(DEV), p2d.to(DEV).requires_grad_(True)
    for d in (3, 16):
        ca = (torch.rand(B, p2d.shape[1], 3 * d, generator=g) * 2 - 1).to(DEV).requires_grad_(True)
        wf = torch.rand(B, RES, RES, d, generator=g).to(DEV)
        for tag, kw in (("", {}), (" params", NONDEFAULT)):
            def run(ca=ca, wf=wf, kw=kw):
                imfeat, improb, _, _ = raster_attr(c3, c2, cn, ca, RES, RES, **kw)
                torch.autograd.grad((imfeat * wf).sum() + (improb * wa).sum(), [c2, ca])
            out[f"attr d={d}{tag}"] = run
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_render_modes.py measures on a CUDA device; none found")
    fns = cases()
    for fn in fns.values():              # warm-up: module loads, allocator, every shape of the timed windows
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(a.rounds):
        for k, fn in fns.items():
            ev[0].record()
            for _ in range(a.iters):
                fn()
            ev[1].record()
            ev[1].synchronize()
            times[k].append(ev[0].elapsed_time(ev[1]) / a.iters)
    res = {"card": card(), "B": B, "res": RES, "faces": 960, "texture": [TEX, TEX + 2], "iters": a.iters,
           "rounds": a.rounds, "ms_per_fwd_bwd": {k: {"median": round(float(np.median(v)), 4),
                                                     "min": round(min(v), 4), "max": round(max(v), 4)}
                                                 for k, v in times.items()}}
    print("card:", res["card"])
    for k, v in res["ms_per_fwd_bwd"].items():
        print(f"  {k:18s} {v['median']:8.3f} ms  ({v['min']:.3f}-{v['max']:.3f})")
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
