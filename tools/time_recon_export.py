"""Timing of the reconstruction export (reconstruction_export.py) on one GPU, at reconstruct.py's defaults for CUB: the
reconstruction network at 256^2 input (random weights: the cost does not depend on them), the 16-ring template, textures
at R 512, the visibility render at 1024^2, views at 512^2.  Prints one JSON line (also written to --out when given):
  1. the exporter's GPU work per batch at B 16 and B 50 (network, vertices_and_pose, index render, texel visibility,
     inverse render of the 1024^2 photo, b3d_recon_texture_pack, the B x 9 view render, b3d_sample_pack, one copy to a
     pinned slot), host time to a device synchronisation;
  2. the b3d_recon_texture_pack launch at B 16 (CUDA events) against its HBM bound, counted from the shapes at 3.35 TB/s;
  3. end-to-end images/s of ReconstructionExporter.export (files written to a temporary directory) with 1, 4 and 16
     writers.
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
R, T, HD = 512, 128, 1024
HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def batch(B, seed):
    """A posed eval batch (X_256, img_1024, scale, translation, rot, ind) on the device."""
    g = torch.Generator().manual_seed(seed)
    return tuple(t.to(DEV) for t in (
        torch.rand(B, 4, 256, 256, generator=g) * 2 - 1, torch.rand(B, 3, HD, HD, generator=g) * 2 - 1,
        0.6 + 0.3 * torch.rand(B, 1, generator=g),
        torch.cat(((torch.rand(B, 2, generator=g) - 0.5) * 0.2, torch.zeros(B, 1)), 1),
        F.normalize(torch.randn(B, 4, generator=g), dim=1), torch.arange(B)))


def time_batches(exp, B, reps):
    from staging import Staging
    b = batch(B, B)
    exp._staging = Staging(DEV, 'timing')

    def one(slot):
        lay, nbytes = exp._device_batch(b, True, True)
        exp._staging.slots[slot][:nbytes].copy_(exp._staging.buffer[:nbytes], non_blocking=True)

    for k in range(2):
        one(k)
    torch.cuda.synchronize()
    t = []
    for k in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        one(k % 2)
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    ms = 1e3 * np.array(t)
    return {'median_ms': float(np.median(ms)), 'min_ms': float(ms.min()), 'max_ms': float(ms.max()),
            'ms_per_image': float(np.median(ms)) / B}


def time_pack(B=16, reps=200):
    from b3d.data import recon_texture_pack
    g = torch.Generator().manual_seed(2)
    vis = (torch.rand(B, T, T, generator=g) < 0.4).to(torch.uint8).to(DEV)
    proj = (torch.rand(B, R, R, 3, generator=g) * 2 - 1).to(DEV)
    alpha = (torch.rand(B, R, R, 1, generator=g) < 0.5).float().to(DEV)
    pred = (torch.rand(B, 3, T, T, generator=g) * 2 - 1).to(DEV)
    tex8 = torch.empty(B, R, R, 3, dtype=torch.uint8, device=DEV)
    src8 = torch.empty(B, R, R, dtype=torch.uint8, device=DEV)
    for _ in range(10):
        recon_texture_pack(vis, proj, alpha, pred, True, tex8, src8)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        recon_texture_pack(vis, proj, alpha, pred, True, tex8, src8)
    e1.record()
    torch.cuda.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / reps
    # every input and output once (a mirrored texel re-reads a row the sample already reads)
    nbytes = vis.numel() + proj.numel() * 4 + alpha.numel() * 4 + pred.numel() * 4 + tex8.numel() + src8.numel()
    bound_us = 1e6 * nbytes / HBM_BYTES_PER_S
    return {'B': B, 'us': us, 'bytes': nbytes, 'hbm_bound_us': bound_us, 'share_of_hbm_bound': bound_us / us}


def time_end_to_end(exp, n, B, writers):
    """One export call over n images in batches of B (the staging pipeline overlaps the GPU work of a batch with the
    writes of the one before)."""
    batches = [batch(B, 100 + k) for k in range(n // B)]
    for k, b in enumerate(batches):
        b[-1].copy_(torch.arange(k * B, (k + 1) * B))
    names = [f'img{i}' for i in range(n)]
    with tempfile.TemporaryDirectory() as d:
        exp.export(batches[:1], names, os.path.join(d, 'warm'), writers=writers, per_index=False)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        exp.export(batches, names, os.path.join(d, 'out'), writers=writers, per_index=False)
        dt = time.perf_counter() - t0
    return {'images_per_s': n / dt, 'seconds': dt, 'images': n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--e2e-images", type=int, default=64)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_recon_export: needs a CUDA device")
    from reconstruction_export import ReconstructionExporter
    from reconstruction_training import ReconTrainer, default_args
    from rendering.mesh_template import MeshTemplate
    from tools.uvsphere import write_uvsphere_obj
    tpl = MeshTemplate(write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16), device=DEV)
    torch.manual_seed(0)
    tr = ReconTrainer(default_args(), tpl, 64, device=DEV)
    exp = ReconstructionExporter(tr, tpl, R)
    tr.generator.eval()
    out = {'card': card(), 'config': dict(template='uvsphere_16rings', export_resolution=R, texture=T, render=HD)}
    with torch.no_grad():
        for B in (16, 50):
            out[f'batch_B{B}'] = time_batches(exp, B, a.reps)
    out['recon_texture_pack'] = time_pack()
    for w in (1, 4, 16):
        out[f'end_to_end_writers{w}'] = time_end_to_end(exp, a.e2e_images, 16, w)
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
