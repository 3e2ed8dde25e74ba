"""Generate tests/golden/samples_reference.npz by EXECUTING the reference's sample export (authoring container only):
    python tests/golden/make_golden_samples.py
The `elif args.save_results:` body of main.py (:836-897) is compiled unmodified from the script's syntax tree, together
with `ModelWrapper` (:449-526) for its 'inference' mode, and run with N = 10 (so the grid's last row is partial) after
np.random.seed(5) / torch.manual_seed(5), with these stand-ins:
  - the generator: wrapper_common.TinyG (class-conditional, latent 8, 8 x 8 texture and displacement map);
  - the dataset: samples_common.PoseSet (poses and classes of 23 samples);
  - the reference's OWN MeshTemplate and Renderer on the 16-ring fixture, with the stand-ins for their kaolin calls of
    make_golden_pseudogt.py (OBJ loading; the ORACLE's rasteriser in place of kaolin's, the one unpinned piece);
  - `.cuda()` = identity; imageio.imwrite capturing the arrays it is given;
  - torchvision.utils.make_grid restated below (padding 0, pad value 0).  torchvision is not installed here, so the grid
    layout is this restatement's, NOT pinned by executing torchvision.
Recorded: the draws (indices, noise, classes), the generator outputs, the object-space and posed vertices, every captured
array (textures, grid) and the .obj / .mtl texts (the files stored compactly: samples_common.pack_files).  The oracle's
face-index buffer of the render is not stored: the tests rasterise the recorded posed vertices with the oracle themselves.  Nothing of the
reference is copied into the repository — only its outputs."""
import ast
import gzip
import math
import os
import pathlib
import sys
import tempfile
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

REF = "/root/reference/code"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, REF)
from oracle import mesh as M                                   # noqa: E402

# ---- stand-ins for kaolin (see make_golden_pseudogt.py), imageio and torchvision --------------------------------------
kal = types.ModuleType("kaolin")
kal.rep = types.ModuleType("kaolin.rep")
face_index = []
written = {}


class Mesh:
    compute_adjacency_info = None


class TriangleMesh(Mesh):
    @classmethod
    def from_obj(cls, path, enable_adjacency=False):
        d = M.load_obj(path)
        m = cls()
        m.vertices, m.faces, m.uvs, m.face_textures = d["vertices"], d["faces"], d["uvs"], d["face_textures"]
        if enable_adjacency:
            m.ff = Mesh.compute_adjacency_info(m.vertices, m.faces)[8]
        return m

    def cuda(self):
        return self


def linear_rasterizer(width, height, p3d, p2d, normalz, attr):
    imfeat, improb, imidx, _ = M.rasterize(p3d, p2d, normalz, attr, height, width)
    face_index.append(imidx)
    return imfeat, improb


def make_grid(tensor, nrow=8, padding=0):
    """torchvision.utils.make_grid for a [n,3,H,W] batch and padding 0: min(nrow, n) columns, ceil(n / columns) rows,
    row-major, unfilled cells 0."""
    assert padding == 0
    n, C, H, W = tensor.shape
    xmaps = min(nrow, n)
    ymaps = int(math.ceil(float(n) / xmaps))
    grid = tensor.new_full((C, H * ymaps, W * xmaps), 0.0)
    for k in range(n):
        y, x = divmod(k, xmaps)
        grid[:, y * H:(y + 1) * H, x * W:(x + 1) * W].copy_(tensor[k])
    return grid


kal.rep.Mesh, kal.rep.TriangleMesh = Mesh, TriangleMesh
mods = {"kaolin": kal, "kaolin.rep": kal.rep}
for n in ("kaolin.graphics", "kaolin.graphics.dib_renderer", "kaolin.graphics.dib_renderer.rasterizer", "kaolin.graphics.dib_renderer.utils",
          "torchvision", "torchvision.models", "torchvision.utils", "imageio"):
    mods[n] = types.ModuleType(n)
mods["kaolin.graphics.dib_renderer.rasterizer"].linear_rasterizer = linear_rasterizer
mods["kaolin.graphics.dib_renderer.utils"].datanormalize = M.datanormalize
mods["torchvision"].models, mods["torchvision"].utils = mods["torchvision.models"], mods["torchvision.utils"]
mods["torchvision.utils"].make_grid = make_grid
mods["imageio"].imwrite = lambda path, arr: written.__setitem__(path, np.array(arr))
sys.modules.update(mods)
torch.Tensor.cuda = lambda self, *a, **k: self                 # D15

from rendering.mesh_template import MeshTemplate               # noqa: E402  (reference)
from rendering.renderer import Renderer                        # noqa: E402  (reference)
from rendering.utils import qrot                               # noqa: E402  (reference)
from utils.losses import GANLoss                               # noqa: E402  (reference)
import samples_common as SC                                    # noqa: E402
import wrapper_common as WC                                    # noqa: E402


def main():
    src = open(os.path.join(REF, "main.py")).read()
    tree = ast.parse(src)
    defs = {n.name: n for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef))}
    block = next(n for n in ast.walk(tree) if isinstance(n, ast.If) and isinstance(n.test, ast.Attribute)
                 and n.test.attr == "save_results" and isinstance(n.body[0], ast.With))
    wrapper = ast.get_source_segment(src, defs["ModelWrapper"]).replace(
        "GANLoss(args.loss, tensor=torch.cuda.FloatTensor).cuda()", "GANLoss(args.loss, tensor=torch.FloatTensor)")
    args = WC.make_args(2, 512)
    args.conditional_class, args.batch_size, args.truncation_sigma, args.weights = True, SC.N, SC.SIGMA, "golden"
    assert args.latent_dim == SC.LATENT
    ns = {"torch": torch, "nn": nn, "math": math, "np": np, "GANLoss": GANLoss, "args": args}
    exec(compile(wrapper, "main.py", "exec"), ns)
    gi, _ = WC.build()
    trainer = ns["ModelWrapper"](gi, None)

    tmp = tempfile.mkdtemp()
    path = os.path.join(tmp, "uvsphere_16rings.obj")
    with gzip.open(os.path.join(HERE, "uvsphere_16rings.obj.gz"), "rb") as s, open(path, "wb") as d:
        d.write(s.read())
    mesh_template = MeshTemplate(path, is_symmetric=True)
    seen = {}
    trainer.generator_running_avg.register_forward_hook(
        lambda m, inp, out: seen.update(noise=inp[0].clone(), c=inp[1].clone(), tex=out[0].clone(), mesh=out[1].clone()))
    get_vertex_positions, forward_renderer = mesh_template.get_vertex_positions, mesh_template.forward_renderer

    def recording_vertices(mesh_map):
        seen["raw"] = get_vertex_positions(mesh_map)
        return seen["raw"]

    def recording_render(renderer, vtx, tex, **kw):
        seen["posed"] = vtx.clone()
        return forward_renderer(renderer, vtx, tex, **kw)
    mesh_template.get_vertex_positions, mesh_template.forward_renderer = recording_vertices, recording_render

    ds = SC.PoseSet()
    ns.update(trainer=trainer, generator_running_avg=trainer.generator_running_avg, mesh_template=mesh_template,
              renderer=Renderer(SC.RENDER, SC.RENDER), train_ds=ds, gpu_ids=[0], qrot=qrot, F=F, os=os, pathlib=pathlib)
    cwd = os.getcwd()
    os.chdir(tmp)
    try:
        np.random.seed(SC.SEED)
        torch.manual_seed(SC.SEED)
        exec(compile(ast.Module(body=block.body, type_ignores=[]), "main.py", "exec"), ns)
    finally:
        os.chdir(cwd)

    out_dir = os.path.join(tmp, "results", "golden")
    assert len(face_index) == 1 and len(written) == SC.N + 1
    objs = [open(os.path.join(out_dir, f"mesh_{i}.obj")).read() for i in range(SC.N)]
    mtls = [open(os.path.join(out_dir, f"mesh_{i}.mtl")).read() for i in range(SC.N)]
    grid = written[os.path.join("results", "golden.png")]
    out = dict(indices=np.asarray(ns["indices"]), noise=seen["noise"].numpy(), classes=seen["c"].numpy(),
               pred_tex=seen["tex"].numpy(), pred_mesh=seen["mesh"].numpy(), vertices=seen["raw"].numpy(),
               posed=seen["posed"].numpy(),
               textures=np.stack([written[os.path.join("results", "golden", f"mesh_{i}.png")] for i in range(SC.N)]),
               **SC.pack_files(objs, mtls, grid))
    o, m, g = SC.unpack_files(out)
    assert o == objs and m == mtls and np.array_equal(g, grid)
    assert torch.equal(ns["noise"], seen["noise"])
    p = os.path.join(HERE, "samples_reference.npz")
    np.savez_compressed(p, **out)
    print("wrote", p, os.path.getsize(p), "bytes; indices", out["indices"], "coverage",
          float((face_index[0] > 0).float().mean()), "grid", grid.shape)


if __name__ == "__main__":
    main()
