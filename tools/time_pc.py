"""Device timing of the point-cloud silhouette kernels at cfg3's size (B 32, N 8000, V 128).  CUDA events around the libb3d
entry points, L2 flushed between iterations, median of 20.  Given a file name, the first run saves its outputs there and a
later run (e.g. of another build) prints its difference to them."""
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "2dimageto3dmodel_b200"))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import b3d  # noqa: E402
from b3d import pointcloud as pc  # noqa: E402

B, N, V = 32, 8000, 128
dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
# points on a noisy sphere surface of radius 0.35 (SURVEY 8d: the realistic collision pattern)
d = torch.nn.functional.normalize(torch.randn(B, N, 3, generator=g), dim=-1)
p = (d * (0.35 + 0.01 * torch.randn(B, N, 1, generator=g))).to(dev).requires_grad_(True)
q = torch.randn(B, 4, generator=g).to(dev).requires_grad_(True)
s = (0.5 + 0.5 * torch.rand(B, 1, generator=g)).to(dev).requires_grad_(True)
w = torch.rand(B, V, V, generator=g).to(dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
rec = {}
ITERS = int(os.environ.get("ITERS", 25))
for it in range(ITERS):
    flush.zero_()
    for t in (p, q, s):
        t.grad = None
    if it >= 5:
        b3d.prof_enable()
    sil = pc.effective_loss(p, q, s, V=V)
    (sil * w).sum().backward()
    if it >= 5:
        for k, v in b3d.prof_disable().items():
            rec.setdefault(k, []).append(sum(v))
print("  ".join(f"{k.replace('b3d_pc_', '')} {statistics.median(v) * 1e3:.1f} us" for k, v in sorted(rec.items())))
out = {"sil": sil.detach().cpu(), "dp": p.grad.cpu(), "dq": q.grad.cpu(), "ds": s.grad.cpu()}
if len(sys.argv) > 1:
    f = sys.argv[1]
    if os.path.exists(f):
        other = torch.load(f)
        print(f"max |difference| to {f}:", {k: float((out[k] - other[k]).abs().max()) for k in out},
              "scale", {k: float(other[k].abs().max()) for k in out})
    else:
        torch.save(out, f)
