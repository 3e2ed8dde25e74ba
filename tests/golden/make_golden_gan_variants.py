"""Generate tests/golden/gan_variants_reference.npz from the REFERENCE's own modules (authoring container only):
    python tests/golden/make_golden_gan_variants.py
Imports models/gan.py and utils/losses.py unmodified from /root/reference/code (they run on CPU), builds G and D for each
configuration of tests/golden/gan_variants_common.py, and stores, under the key prefix "<config>/":
  - the initial state dicts of G and D (names, shapes, fp64 sums: the CUDA modules must build the same tensors);
  - one generator step and one discriminator step in training mode (probes, losses, per-parameter gradient norms), as
    make_golden_gan.py does for the default configuration;
  - an eval-mode generator forward after the two steps."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, "/root/reference/code")
import gan_common as GC                                     # noqa: E402
import gan_variants_common as GV                            # noqa: E402
from models import gan as ref_gan                           # noqa: E402  (reference)
from utils.losses import GANLoss                            # noqa: E402  (reference)


def make(name, out):
    torch.set_num_threads(8)
    args, G, D = GV.build(ref_gan, name)
    nd = args.num_discriminators
    k = name + "/"
    for tag, m in (("g", G), ("d", D)):
        names, shapes, sums = GV.state_summary(m)
        out[k + tag + "_state_names"] = np.array(names)
        out[k + tag + "_state_shapes"] = np.array(shapes)
        out[k + tag + "_state_sums"] = np.array(sums)
    G.train(); D.train()
    crit = GANLoss('hinge', tensor=torch.FloatTensor)
    z, c, alpha, tex, mesh = GC.inputs(args, B=GV.B)
    # ---- generator step
    loss, pred_tex, pred_mesh, dout, mask = GC.g_step(G, D, crit, z, c, alpha)
    loss.mean().backward()
    out[k + "g_loss"] = loss.detach().numpy()
    out[k + "tex_probe"] = pred_tex.detach()[:, :, ::16, ::16].numpy()
    out[k + "tex_sum"] = np.float64(pred_tex.detach().double().sum())
    out[k + "mesh"] = pred_mesh.detach().numpy()
    for i in range(nd):
        out[k + f"d_out{i}"] = dout[i].detach().numpy()
    names = [n for n, p in G.named_parameters() if p.grad is not None]
    out[k + "g_grad_names"] = np.array(names)
    out[k + "g_grad_norms"] = np.array([float(dict(G.named_parameters())[n].grad.norm()) for n in names])
    G.zero_grad(); D.zero_grad()
    # ---- discriminator step
    lf, lr, dout = GC.d_step(G, D, crit, z, c, alpha, tex, mesh)
    (lf.mean() + lr.mean()).backward()
    out[k + "d_loss_fake"], out[k + "d_loss_real"] = lf.detach().numpy(), lr.detach().numpy()
    for i in range(nd):
        out[k + f"dd_out{i}"] = dout[i].detach().numpy()
    names = [n for n, p in D.named_parameters() if p.grad is not None]
    out[k + "d_grad_names"] = np.array(names)
    out[k + "d_grad_norms"] = np.array([float(dict(D.named_parameters())[n].grad.norm()) for n in names])
    # ---- eval-mode generator forward (running statistics for batch norms, instance statistics for instance norms)
    G.eval()
    with torch.no_grad():
        et, em = G(z, c)
    out[k + "eval_tex_probe"] = et[:, :, ::16, ::16].numpy()
    out[k + "eval_mesh"] = em.numpy()
    print(name, "g_loss", float(loss), "d losses", float(lf), float(lr), flush=True)


if __name__ == "__main__":
    out = {}
    for name in GV.CONFIGS:
        make(name, out)
    path = os.path.join(HERE, "gan_variants_reference.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")
