"""Timing of the sample export (sample_export.py) on one GPU, at the reference's defaults for CUB: the 512^2 generator of the
shipped weights (random weights: the cost does not depend on them), the 16-ring template, renders at 512^2.  Prints one
JSON line (also written to --out when given):
  1. per batch at B 16, alternated in one run: the exporter's GPU work (generator, vertices_and_pose, render,
     b3d_sample_pack, the vertex rows, one copy to a pinned slot) against the reference's composition on the same noise
     (main.py:867-893: get_vertex_positions, the Y/Z swap, export_obj's per-sample texture bytes and .cpu(), qrot / scale /
     translate / flip, the hard-mask render, the background fill, permute, / 2 + 0.5, avg_pool2d, make_grid's copies,
     * 255, clamp, .cpu().byte()), host time to a device synchronisation;
  2. the b3d_sample_pack launch (CUDA events) against its HBM bound, counted from the shapes at 3.35 TB/s;
  3. end-to-end samples/s of SampleExporter.export (files written to a temporary directory) with 1, 4 and 16 writers.
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
import torch.nn.functional as F   # noqa: E402

DEV = "cuda:0"
B, RES = 16, 512
HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


class Poses:
    """A CUB-sized pose table with class labels (what SampleExporter reads from the dataset)."""

    def __init__(self, n=5964, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.data = {'scale': 0.6 + 0.3 * torch.rand(n, 1, generator=g),
                     'translation': torch.cat(((torch.rand(n, 2, generator=g) - 0.5) * 0.2, torch.zeros(n, 1)), 1),
                     'rotation': F.normalize(torch.randn(n, 4, generator=g), dim=1)}
        self.classes = [np.array([i % 200]) for i in range(n)]

    def __len__(self):
        return len(self.classes)


def reference_composition(exp, noise, c, scale, trans, rot):
    """main.py:865-893 on the CUDA renderer, without the file writes."""
    from rendering.utils import qrot
    with torch.no_grad():
        pred_tex, mesh_map, _ = exp.generator(noise, c, None, return_attention=True)
        vtx = exp.tpl.get_vertex_positions(mesh_map)
        vtx_obj = vtx.clone()
        vtx_obj[..., :] = vtx_obj[..., [0, 2, 1]]
        texs = [((pred_tex[i] / 2 + 0.5).permute(1, 2, 0) * 255).clamp(0, 255).cpu().byte().numpy()
                for i in range(noise.shape[0])]
        verts = [v.cpu().numpy() for v in vtx_obj]
        vtx = qrot(rot, scale.unsqueeze(-1) * vtx) + trans.unsqueeze(1)
        vtx = vtx * torch.tensor([1.0, -1.0, -1.0], device=vtx.device)
        image_pred, alpha_pred = exp.tpl.forward_renderer(exp.renderer, vtx, pred_tex, return_hardmask=True)
        image_pred[alpha_pred.expand_as(image_pred) == 0] = 1
        image_pred = F.avg_pool2d(image_pred.permute(0, 3, 1, 2) / 2 + 0.5, 2)
        grid = torch.zeros(3, 2 * 256, 8 * 256, device=DEV)            # make_grid(nrow=8, padding=0) of 16 tiles
        for k in range(noise.shape[0]):
            grid[:, (k // 8) * 256:(k // 8 + 1) * 256, (k % 8) * 256:(k % 8 + 1) * 256].copy_(image_pred[k])
        grid = (grid.permute(1, 2, 0) * 255).clamp(0, 255).cpu().byte().numpy()
    return texs, verts, grid


def time_batches(exp, reps):
    from staging import Staging
    ds = exp.ds
    g = torch.Generator().manual_seed(1)
    idx = torch.randperm(len(ds), generator=g)[:B]
    scale = ds.data['scale'][idx].to(DEV)
    trans, rot = ds.data['translation'][idx].to(DEV), ds.data['rotation'][idx].to(DEV)
    c = torch.as_tensor(np.stack([ds.classes[i] for i in idx.tolist()])).to(DEV)
    noise = torch.randn(B, 64, generator=g).clamp(-0.25, 0.25).to(DEV)
    exp._staging = Staging(DEV, 'timing')

    def exporter(slot):
        lay, nbytes = exp._device_batch(noise, c, scale, trans, rot)
        exp._staging.slots[slot][:nbytes].copy_(exp._staging.buffer[:nbytes], non_blocking=True)

    for k in range(2):                                          # warm-up of both paths
        exporter(k)
        reference_composition(exp, noise, c, scale, trans, rot)
    torch.cuda.synchronize()
    t = {'exporter': [], 'reference': []}
    for k in range(reps):
        for name in (('exporter', 'reference') if k % 2 == 0 else ('reference', 'exporter')):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if name == 'exporter':
                exporter(k % 2)
            else:
                reference_composition(exp, noise, c, scale, trans, rot)
            torch.cuda.synchronize()
            t[name].append(time.perf_counter() - t0)
    return {k: {'median_ms': 1e3 * float(np.median(v)), 'min_ms': 1e3 * float(np.min(v)), 'max_ms': 1e3 * float(np.max(v))}
            for k, v in t.items()}


def time_pack(reps=200):
    from b3d.data import sample_pack
    g = torch.Generator().manual_seed(2)
    image = (torch.rand(B, RES, RES, 3, generator=g) * 2 - 1).to(DEV)
    imidx = torch.randint(0, 900, (B, RES, RES), generator=g, dtype=torch.int32).to(DEV)
    tex = (torch.rand(B, 3, RES, RES, generator=g) * 2 - 1).to(DEV)
    tiles = torch.empty(B, RES // 2, RES // 2, 3, dtype=torch.uint8, device=DEV)
    tex8 = torch.empty(B, RES, RES, 3, dtype=torch.uint8, device=DEV)
    for _ in range(10):
        sample_pack(image, imidx, tex, tiles, tex8)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        sample_pack(image, imidx, tex, tiles, tex8)
    e1.record()
    torch.cuda.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / reps
    nbytes = image.numel() * 4 + imidx.numel() * 4 + tex.numel() * 4 + tiles.numel() + tex8.numel()
    bound_us = 1e6 * nbytes / HBM_BYTES_PER_S
    return {'us': us, 'bytes': nbytes, 'hbm_bound_us': bound_us, 'share_of_hbm_bound': bound_us / us}


def time_end_to_end(exp, n, writers):
    with tempfile.TemporaryDirectory() as d:
        exp.export(os.path.join(d, 'warm'), os.path.join(d, 'warm.png'), B, B, seed=0, writers=writers)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        exp.export(os.path.join(d, 'out'), os.path.join(d, 'grid.png'), n, B, seed=1, writers=writers)
        dt = time.perf_counter() - t0
    return {'samples_per_s': n / dt, 'seconds': dt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--e2e-samples", type=int, default=64)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_samples: needs a CUDA device")
    import bench
    from gan_training import GANTrainer
    from rendering.mesh_template import MeshTemplate
    from sample_export import SampleExporter
    from tools.uvsphere import write_uvsphere_obj
    tpl = MeshTemplate(write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16), device=DEV)
    torch.manual_seed(0)
    args = bench.gan_args(RES, 3)
    tr = GANTrainer(args, mesh_template=tpl, device=DEV)
    exp = SampleExporter(tr.trainer.generator_running_avg, tpl, Poses(), 0.25, latent_dim=args.latent_dim)
    exp.generator.eval()
    out = {'card': card(), 'config': dict(template='uvsphere_16rings', texture=RES, render=RES, batch=B)}
    out['batch_B16'] = time_batches(exp, a.reps)
    out['sample_pack_B16'] = time_pack()
    for w in (1, 4, 16):
        out[f'end_to_end_writers{w}'] = time_end_to_end(exp, a.e2e_samples, w)
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
