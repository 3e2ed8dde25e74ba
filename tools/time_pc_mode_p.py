"""Fused against dense mode-P effective loss (paper semantics), forward + backward, in one job and alternated.

For each shape: CUDA events around forward + backward of `effective_loss(mode="P")` (the fused entry points) and of
`effective_loss_dense(mode="P")` (one stand-alone kernel per stage), L2 flushed before every iteration, median of
--iters after --warmup; peak `torch.cuda.max_memory_allocated` of each path above what the inputs hold; the grid bytes each
path moves, counted from shapes, and the time HBM needs for them at 3.35 TB/s (the H100 SXM data-sheet figure).
Prints one JSON line per shape and a summary line with the GPU name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "2dimageto3dmodel_b200"))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from b3d.pointcloud import effective_loss, effective_loss_dense, smoothing_taps  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
# full-grid transfers (one read or one write of B V^3 fp32) per forward + backward, from the launches:
#   fused  fwd: zero A, x/y blur (read A, write B), z blur + ray march (read B) = 4;
#          bwd: column adjoints (read B, write B), x/y adjoints (read B, read A, write A) = 5
#   dense  fwd: zero, clone (2), clamp (2), three blurs (6), scale/clamp (2), termination (1) = 14;
#          bwd: termination adjoint (reads the grid twice, writes and re-reads T: 5), scale adjoint (3), three transposed
#          blurs (6), clone (2), clamp mask (3) = 19
GRID_PASSES = {"fused": 9, "dense": 33}


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shapes", default="16x8000x128,16x8000x64,64x8000x128", help="BxNxV,...")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    taps = smoothing_taps(3.0, 21, "P")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    paths = {"fused": effective_loss, "dense": effective_loss_dense}
    for shape in args.shapes.split(","):
        B, N, V = (int(v) for v in shape.split("x"))
        g = torch.Generator().manual_seed(0)
        d = torch.nn.functional.normalize(torch.randn(B, N, 3, generator=g), dim=-1)
        p = (d * (0.35 + 0.01 * torch.randn(B, N, 1, generator=g))).to(dev).requires_grad_(True)
        q = torch.randn(B, 4, generator=g).to(dev).requires_grad_(True)
        s = (0.5 + 0.5 * torch.rand(B, 1, generator=g)).to(dev).requires_grad_(True)
        w = torch.rand(B, V, V, generator=g).to(dev)
        times = {k: [] for k in paths}
        peak = {}
        outs = {}
        for it in range(args.warmup + args.iters):
            for name, fn in paths.items():          # alternated within every iteration
                for t in (p, q, s):
                    t.grad = None
                flush.zero_()
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                sil = fn(p, q, s, V=V, taps=taps, mode="P")
                (sil * w).sum().backward()
                e1.record()
                torch.cuda.synchronize()
                if it >= args.warmup:
                    times[name].append(e0.elapsed_time(e1))
                peak[name] = max(peak.get(name, 0), torch.cuda.max_memory_allocated() - base)
                outs[name] = [sil.detach().clone()] + [t.grad.clone() for t in (p, q, s)]
                del sil
        diff = {k: float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
                for k, a, b in zip(["sil", "dp", "dq", "ds"], outs["fused"], outs["dense"])}
        grid = B * V ** 3 * 4
        rec = {"B": B, "N": N, "V": V}
        for name in paths:
            moved = GRID_PASSES[name] * grid
            rec[name] = {"ms_median": statistics.median(times[name]), "ms_min": min(times[name]),
                         "ms_max": max(times[name]), "peak_mb": peak[name] / 2 ** 20,
                         "grid_gb_moved": moved / 1e9, "hbm_bound_ms": moved / HBM_BYTES_PER_S * 1e3}
        rec["speedup"] = rec["dense"]["ms_median"] / rec["fused"]["ms_median"]
        rec["max_rel_diff_fused_vs_dense"] = diff
        print(json.dumps(rec), flush=True)
        del p, q, s, w, outs
        torch.cuda.empty_cache()
    print(json.dumps({"gpu": gpu_name(), "iters": args.iters, "warmup": args.warmup}))


if __name__ == "__main__":
    main()
