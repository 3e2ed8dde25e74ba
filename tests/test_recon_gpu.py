"""models.reconstruction.ReconstructionNetwork on the wgmma conv kernels against golden vectors produced by the
reference's own module on the CPU (tests/golden/make_golden_recon.py): same seed -> same weights, same inputs, one
training-mode forward + backward (batch statistics, stride-2 3x3 / 5x5 encoder convs, ResBlocks, thin 3-channel heads).

Tolerance: the golden is exact fp32, the tensor cores compute in tf32.  Emulating tf32 rounding of every convolution
operand in the reference itself (authoring container) moves the texture by 1.8e-2 of its range, the displacement map by
5e-3 and per-parameter gradient norms by < 3 % — the limits below are ~2.5x that."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import recon_common as RC          # noqa: E402

pytestmark = pytest.mark.gpu


def close(a, ref, tol):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    err = float(np.abs(a - ref).max())
    lim = tol * max(float(np.abs(ref).max()), 1e-6)
    assert err <= lim, (err, lim)


def test_reconstruction_network_matches_reference_golden():
    from models import reconstruction
    d = np.load(os.path.join(GOLDEN, "recon_reference.npz"))
    net = RC.build(reconstruction).cuda().train()
    x, w_tex, w_mesh = [t.cuda() for t in RC.inputs()]
    tex, mesh_map = net(x)
    assert tex.shape == (8, 3, 128, 128) and mesh_map.shape == (8, 3, 32, 32)
    RC.loss_of(tex, mesh_map, w_tex, w_mesh).backward()
    close(tex[:, :, ::8, ::8], d["tex_probe"], 5e-2)
    assert abs(float(tex.double().sum()) - float(d["tex_sum"])) < 2e-2 * tex.numel() ** 0.5 * 5
    close(mesh_map, d["mesh_map"], 2e-2)
    for t in (tex, mesh_map):                               # symmetric output: mirrored about the seam at a quarter width
        q = t.shape[3] // 4
        assert torch.equal(t[..., :q], t[..., q:2 * q].flip(3)) and torch.equal(t[..., 3 * q:], t[..., 2 * q:3 * q].flip(3))
    params = dict(net.named_parameters())
    floor = 5e-3 * float(d["grad_norms"].max())
    for name, ref in zip(d["grad_names"], d["grad_norms"]):
        got = float(params[str(name)].grad.norm())
        assert abs(got - ref) <= 8e-2 * ref + floor, (str(name), got, ref)
    close(net.bn4e.running_mean, d["bn4e_mean"], 2e-2)
    close(net.blk2.bn2.running_var, d["bn_blk2_var"], 5e-2)


def test_reconstruction_network_has_no_cpu_fallback():
    from b3d import B3DError
    from models import reconstruction
    net = reconstruction.ReconstructionNetwork(symmetric=True, texture_res=64)
    with pytest.raises(B3DError):
        net(torch.zeros(2, 4, 256, 256))
