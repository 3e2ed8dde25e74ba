"""Timing of the pseudo-ground-truth export (pseudo_gt_export.py) on one GPU, at the reference's defaults: CUB's 16-ring
template, texture 128, loader sizes [256, 299, 1024], pseudo-GT resolution R 512, the full 2048-d Inception network (random
weights: the cost does not depend on them).  Prints one JSON line (also written to --out when given):
  1. per batch at B 10 and B 50, alternated in one run: the exporter's GPU work (network, pose, unshaded render,
     b3d_texel_visibility, Inception features, inverse render, b3d_pseudogt_pack, one copy to a pinned slot) against the
     reference's construction (shaded render + autograd visibility, visibility_to_mask, mask, permute, .half(), one .cpu()
     per tensor per sample), host time to a device synchronisation;
  2. b3d_texel_visibility against the texture adjoint of b3d_mesh_render_bwd on the same render (CUDA events);
  3. end-to-end images/s of PseudoGTExporter.export (records compressed and written to a temporary directory) with 1, 4
     and 16 writer threads.
The card's name, power limit and SM clock limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "2dimageto3dmodel_b200"))
sys.path.insert(0, ROOT)

import numpy as np   # noqa: E402
import torch         # noqa: E402

DEV = "cuda:0"
R, RENDER, TEX = 512, 1024, 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def random_inception():
    import math
    from utils.inception import InceptionV3
    net = InceptionV3([3], weights=None)
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, torch.nn.Conv2d):
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * math.sqrt(2.0 / m.weight[0].numel()))
    return net


def batches(n, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for k in range(n):
        out.append(tuple(t.to(DEV) for t in (
            torch.rand(B, 4, 256, 256, generator=g) * 2 - 1, torch.rand(B, 3, 299, 299, generator=g) * 2 - 1,
            torch.rand(B, 3, RENDER, RENDER, generator=g) * 2 - 1, 0.6 + 0.3 * torch.rand(B, 1, generator=g),
            torch.cat(((torch.rand(B, 2, generator=g) - 0.5) * 0.2, torch.zeros(B, 1)), 1),
            torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=1), torch.arange(k * B, (k + 1) * B))))
    return out


def reference_construction(exp, batch):
    """run_reconstruction.py:544-603 on the CUDA renderer, without the file writes."""
    import torch.nn.functional as F
    from data.pseudo_gt import make_record, visibility_to_mask
    from rendering.inverse_renderer import texel_visibility
    from utils.fid import forward_inception_features
    X, img299, hd, scale, trans, rot, ind = batch
    with torch.no_grad():
        pred_tex, mesh_map = exp.trainer.generator(X)
        vtx = exp._pose(mesh_map, scale, trans, rot, ind)
    vis, _, _ = texel_visibility(exp.tpl, exp._renderer, vtx, pred_tex)
    with torch.no_grad():
        forward_inception_features(exp.inception, img299 / 2 + 0.5)
        inv_tex, inv_alpha = exp.inverse_renderer(vtx, hd)
        mask = visibility_to_mask(vis, R)
        inv_tex = (inv_tex * mask).permute(0, 3, 1, 2).half().cpu()
        inv_alpha = (inv_alpha * mask).permute(0, 3, 1, 2).half().cpu()
        return [make_record(mesh_map[i], inv_tex[i], inv_alpha[i], img299[i]) for i in range(X.shape[0])]


def exporter_batch(exp, batch, slot):
    lay, nbytes = exp._device_batch(batch, None)
    exp._slots[slot][:nbytes].copy_(exp._staging[:nbytes], non_blocking=True)


def time_batches(exp, B, reps):
    bs = batches(2, B, seed=B)
    exp._reset()
    for b in bs:                                    # warm-up of both paths (allocator, module loads, staging)
        exporter_batch(exp, b, 0)
        reference_construction(exp, b)
    torch.cuda.synchronize()
    t = {'exporter': [], 'reference': []}
    for k in range(reps):
        for name in (('exporter', 'reference') if k % 2 == 0 else ('reference', 'exporter')):
            b = bs[k % 2]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if name == 'exporter':
                exporter_batch(exp, b, k % 2)
            else:
                reference_construction(exp, b)
            torch.cuda.synchronize()
            t[name].append(time.perf_counter() - t0)
    return {k: {'median_ms': 1e3 * float(np.median(v)), 'min_ms': 1e3 * float(np.min(v)), 'max_ms': 1e3 * float(np.max(v))}
            for k, v in t.items()}


def time_visibility(exp, B, reps=20):
    from b3d import check, lib, ptr, stream_ptr
    from b3d.mesh import face_setup, render_indices, texel_visibility
    X, img299, hd, scale, trans, rot, ind = batches(1, B, seed=7)[0]
    with torch.no_grad():
        pred_tex, mesh_map = exp.trainer.generator(X)
        vtx = exp._pose(mesh_map, scale, trans, rot, ind)
        uvs, tex = exp.tpl.adjust_uv_and_texture(pred_tex)
    tex = tex.contiguous()
    Th, Tw = tex.shape[2], tex.shape[3]
    faces, ft = exp.tpl.mesh.faces, exp.tpl.mesh.face_textures
    imidx, imwei, fuv = render_indices(vtx, faces, uvs, ft, RENDER, RENDER)
    fgeo, fuv2, _ = face_setup(vtx, faces, uvs, ft)
    F = fgeo.shape[1]
    ones = torch.ones(B, RENDER, RENDER, 3, device=DEV)
    dfp, dfuv = torch.empty(B, F, 6, device=DEV), torch.empty(B, F, 6, device=DEV)
    dtex = torch.empty_like(tex)
    out = torch.empty(B, Th, Tw - 2, dtype=torch.uint8, device=DEV)
    words = torch.empty(B, (Th * (Tw - 2) + 31) // 32, dtype=torch.int32, device=DEV)

    def vis():
        texel_visibility(imidx, imwei, fuv, Th, Tw, True, out=out, words=words)

    def adjoint():
        check(lib.b3d_mesh_render_bwd(ptr(fgeo), ptr(fuv2), ptr(tex), 0, B, F, RENDER, RENDER, Th, Tw, ptr(imidx),
                                      ptr(imwei), ptr(ones), None, ptr(dfp), ptr(dfuv), ptr(dtex), stream_ptr(fgeo)))

    res = {}
    for name, fn in (('texel_visibility', vis), ('render_bwd_texture_adjoint', adjoint)):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res[name + '_us'] = 1e3 * e0.elapsed_time(e1) / reps
    return res


def time_end_to_end(exp, B, n_batches, writers):
    bs = batches(n_batches, B, seed=11)
    paths = [f"img{i}.jpg" for i in range(n_batches * B)]
    with tempfile.TemporaryDirectory() as d:
        exp.export(bs[:1], paths, os.path.join(d, 'warm'), 'cub', writers=writers)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        exp.export(bs, paths, os.path.join(d, 'cub'), 'cub', writers=writers)
        dt = time.perf_counter() - t0
        size = sum(os.path.getsize(os.path.join(d, 'cub', f'pseudogt_{R}x{R}', f))
                   for f in os.listdir(os.path.join(d, 'cub', f'pseudogt_{R}x{R}')))
    return {'images_per_s': n_batches * B / dt, 'seconds': dt, 'mean_record_bytes': size / (n_batches * B)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--e2e-batches", type=int, default=4)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_pseudogt: needs a CUDA device")
    from pseudo_gt_export import PseudoGTExporter
    from reconstruction_training import ReconTrainer, default_args
    from rendering.mesh_template import MeshTemplate
    from rendering.renderer import Renderer
    from tools.uvsphere import write_uvsphere_obj
    tpl = MeshTemplate(write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16), device=DEV)
    torch.manual_seed(0)
    tr = ReconTrainer(default_args(texture_resolution=TEX), tpl, 5964, device=DEV)
    with torch.no_grad():
        tr.dataset_params.ds_translation.normal_(0, 0.02)
        tr.dataset_params.ds_scale.normal_(0, 0.02)
    exp = PseudoGTExporter(tr, tpl, R, inception=random_inception())
    exp._renderer = Renderer(RENDER, RENDER)
    tr.generator.eval()
    out = {'card': card(), 'config': dict(template='uvsphere_16rings', texture=TEX, render=RENDER, R=R,
                                          img_size=[256, 299, RENDER])}
    for B in (10, 50):
        out[f'batch_B{B}'] = time_batches(exp, B, a.reps)
        out[f'visibility_B{B}'] = time_visibility(exp, B)
    for w in (1, 4, 16):
        out[f'end_to_end_B50_writers{w}'] = time_end_to_end(exp, 50, a.e2e_batches, w)
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
