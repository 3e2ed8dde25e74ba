"""Timing of the GAN option variants on one GPU at cfg3's size (B 32, 256², two discriminators).  Prints one JSON line
(also written to --out when given):
  1. per configuration of tests/golden/gan_variants_common.py (its norm_g / norm_d / symmetric options at this size): one
     generator step plus two discriminator steps of GANTrainer, the fused generator against the module path
     (disable_fusion), alternated windows timed with CUDA events after warm-up, median over the windows;
  2. per discriminator instance-norm layer of the D step (N 64): the fused glue (b3d.ew.in_act_pad: per-sample sums,
     prepare, normalise + affine + LeakyReLU + circular pad) against the torch composition (InstanceNorm2d -> F.leaky_relu
     -> pad_x) on the same conv outputs, forward and forward + backward, with the forward's HBM bound (y read once, the
     padded output written once, over 3.35 TB/s).
The card's name, power limit and SM clock limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "2dimageto3dmodel_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, ROOT)

import torch         # noqa: E402

HBM_BYTES_PER_S = 3.35e12     # H100 SXM data sheet
D_LAYERS = [("d1.bn2", 128, 128, 128, 1), ("d1.bn3", 256, 64, 64, 1), ("d1.bn4", 512, 32, 32, 2), ("d2.bn2", 128, 16, 16, 1),
            ("d2.bn3", 256, 8, 8, 2)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def window(fn, k):
    """Device time of k calls of fn, in ms per call."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(k):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / k


def alternate(fns, k, windows, warmup):
    """{name: median ms} of alternated windows of each function."""
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    times = {n: [] for n in fns}
    for _ in range(windows):
        for n, fn in fns.items():
            times[n].append(window(fn, k))
    return {n: sorted(t)[len(t) // 2] for n, t in times.items()}


def time_configs(B, windows, k):
    import bench
    import gan_common as GC
    import gan_variants_common as GV
    from gan_training import GANTrainer
    dev = torch.device("cuda")
    out = {}
    for name, cfg in GV.CONFIGS.items():
        args = bench.gan_args(256, 2)
        args.norm_g, args.norm_d, args.symmetric_g = cfg["norm_g"], cfg["norm_d"], cfg["symmetric"]
        torch.manual_seed(4321)
        tr = GANTrainer(args, mesh_template=None, device=dev)
        bs = []
        for i in range(3):
            z, c, alpha, tex, mesh = (t.to(dev) for t in GC.inputs(GC.make_args(256, 2), B=B, seed=100 + i))
            bs.append(dict(X_tex=tex, X_alpha=alpha, X_mesh=mesh, C=c, noise=z))
        G = tr.trainer.generator

        def step(fused):
            G.disable_fusion = not fused
            tr.g_step(bs[0]["X_alpha"], bs[0]["C"], bs[0]["noise"])
            for b in bs[1:]:
                tr.d_step(b["X_tex"], b["X_alpha"], b["X_mesh"], b["C"], b["noise"])
        med = alternate({"fused": lambda: step(True), "module": lambda: step(False)}, k, windows, 2)
        out[name] = dict(norm_g=cfg["norm_g"], norm_d=cfg["norm_d"], symmetric=cfg["symmetric"],
                         fused_ms=round(med["fused"], 3), module_ms=round(med["module"], 3),
                         speedup=round(med["module"] / med["fused"], 3))
        print(name, out[name], flush=True)
        del tr, G, bs
        torch.cuda.empty_cache()
    return out


def time_layers(N, windows, k):
    import torch.nn.functional as F
    from b3d.ew import CIRCULAR, in_act_pad, pad_x
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    out = {}
    for name, C, H, W, pad in D_LAYERS:
        y = torch.randn(N, H, W, C, device=dev, generator=g).permute(0, 3, 1, 2).requires_grad_(True)
        norm = torch.nn.InstanceNorm2d(C, affine=True).to(dev)
        gout = torch.randn(N, H, W + 2 * pad, C, device=dev, generator=g).permute(0, 3, 1, 2)
        fused = lambda: in_act_pad(y, norm, pad, CIRCULAR)
        torch_ = lambda: pad_x(F.leaky_relu(norm(y), 0.2), pad, CIRCULAR)
        fwd = alternate({"fused": fused, "torch": torch_}, k, windows, 3)
        both = alternate({"fused": lambda: fused().backward(gout), "torch": lambda: torch_().backward(gout)}, k, windows, 3)
        bytes_fwd = 4 * N * H * C * (W + (W + 2 * pad))
        bound_us = bytes_fwd / HBM_BYTES_PER_S * 1e6
        out[name] = dict(shape=[N, C, H, W], pad=pad, fused_fwd_us=round(1e3 * fwd["fused"], 1),
                         torch_fwd_us=round(1e3 * fwd["torch"], 1), fwd_hbm_bound_us=round(bound_us, 1),
                         fused_fwd_share_of_bound=round(bound_us / (1e3 * fwd["fused"]), 3),
                         fused_fwd_bwd_us=round(1e3 * both["fused"], 1), torch_fwd_bwd_us=round(1e3 * both["torch"], 1))
        print(name, out[name], flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_gan_variants: needs a CUDA device (nothing is measured on the host)")
    res = {"card": card(), "batch": a.batch, "resolution": 256, "discriminators": 2,
           "configs": time_configs(a.batch, a.windows, 3), "d_layers": time_layers(2 * a.batch, a.windows, 20)}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
