"""The reconstruction validation pass, turntable render and L1 criterion on the CUDA path (H100):
  * the fused L1 + IoU kernel against torch on real renders, ties included, and the MSE entry points on the same inputs;
  * models.reconstruction in eval mode (running statistics; the decoder's fused bn_act_pad) against the reference's
    eval-mode forward (tests/golden/recon_eval_reference.npz, tolerances of test_recon_gpu.py: tf32);
  * ReconTrainer.evaluate against a hand composition of the same pass, and one batch of 8 against two batches of 4;
  * one loss='l1' training step against the same step with the loss computed by torch;
  * render_multiview against direct renders of each view."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN
from oracle import mesh as OM

sys.path.insert(0, GOLDEN)
import recon_common as RC           # noqa: E402
import recon_eval_common as RE      # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
R = 256


@pytest.fixture(scope="module")
def tpl31():
    from rendering.mesh_template import MeshTemplate
    from tools.uvsphere import write_uvsphere_obj
    return MeshTemplate(write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_31rings.obj"), rings=31), device=DEV)


def disk_batch(B, seed, dataset_size=4722):
    """RGBA targets with a disk alpha and poses in the ranges of the P3D pose metadata (as bench.py's cfg4 inputs)."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, R), torch.linspace(-1, 1, R), indexing="ij")
    disk = ((yy * yy + xx * xx) < 0.45).float()
    X = torch.rand(B, 4, R, R, generator=g) * 2 - 1
    X[:, 3] = disk
    X[:, :3] *= disk
    s = 0.55 + 0.3 * torch.rand(B, 1, generator=g)
    t = (torch.rand(B, 3, generator=g) - 0.5) * 0.3
    q = F.normalize(torch.randn(B, 4, generator=g), dim=-1)
    idx = torch.randint(0, 2 * dataset_size, (B,), generator=g)
    return [v.to(DEV) for v in (X, s, t, q, idx)]


def torch_criterion(loss):
    def fn(image, alpha, X_real):
        X_fake = torch.cat((image, alpha), dim=3).permute(0, 3, 1, 2)
        return (F.l1_loss if loss == "l1" else F.mse_loss)(X_fake, X_real), OM.mean_iou(X_fake[:, 3], X_real[:, 3])
    return fn


# ------------------------------------------------------------------------------------------------ the loss kernels
def test_l1_kernel_matches_torch_with_ties(tpl31):
    from b3d.mesh import _RgbaLoss, rgba_l1_iou, rgba_mse_iou
    from rendering.renderer import Renderer
    B = 8
    g = torch.Generator().manual_seed(5)
    mm = (torch.randn(B, 3, 32, 32, generator=g) * 0.05).to(DEV)
    tex = (torch.rand(B, 3, 128, 128, generator=g) * 2 - 1).to(DEV)
    X, s, t, q, _ = disk_batch(B, 7)
    with torch.no_grad():
        _, vtx = tpl31.vertices_and_pose(mm, s, t, q)
        image, alpha = tpl31.forward_renderer(Renderer(R, R), vtx, tex)
    X[:, :3, 100:140, 60:120] = image.permute(0, 3, 1, 2)[:, :, 100:140, 60:120]      # a block of exact ties
    X[:, 3, 100:140, 60:120] = alpha[..., 0][:, 100:140, 60:120]
    X_fake = torch.cat((image, alpha), dim=3).permute(0, 3, 1, 2)
    d = X_fake - X
    assert int((d == 0).sum()) > 100_000 and bool((alpha == 0).any())     # the block + background pixels

    ref = float(F.l1_loss(X_fake.double(), X.double()))
    loss, counts = _RgbaLoss.apply(image, alpha, X, "l1")
    assert abs(float(loss) - ref) <= 1e-5 * ref
    pa, pt = X_fake[:, 3] > 0.5, X[:, 3] > 0.5
    exp_counts = torch.stack(((pa & pt).sum(dim=(1, 2)), (pa | pt).sum(dim=(1, 2))), dim=1).int()
    assert torch.equal(counts, exp_counts)

    gup = 0.7
    i1, a1 = image.clone().requires_grad_(True), alpha.clone().requires_grad_(True)
    l1, miou = rgba_l1_iou(i1, a1, X)
    assert float(miou) == float(OM.mean_iou(X_fake[:, 3], X[:, 3]))
    gi, ga = torch.autograd.grad(l1 * gup, [i1, a1])
    i2, a2 = image.clone().requires_grad_(True), alpha.clone().requires_grad_(True)
    ri, ra = torch.autograd.grad(F.l1_loss(torch.cat((i2, a2), dim=3).permute(0, 3, 1, 2), X) * gup, [i2, a2])
    mag = np.float32(gup) / np.float32(X.numel())
    for got, want in ((gi, ri), (ga, ra)):
        got, want = got.cpu().numpy(), want.cpu().numpy()
        assert np.array_equal(np.sign(got), np.sign(want))                    # identical signs and identical zeros
        nz = want != 0
        assert np.abs(np.abs(got[nz]) - mag).max() <= np.spacing(mag)      # |g| = g_up / n within 1 ulp
        assert np.abs(np.abs(want[nz]) - mag).max() <= np.spacing(mag)
    assert int((ga == 0).sum()) > 0 and int((gi == 0).sum()) > 0

    # the MSE entry points, same inputs: the shared template keeps their values
    i3, a3 = image.clone().requires_grad_(True), alpha.clone().requires_grad_(True)
    lm, miou_m = rgba_mse_iou(i3, a3, X)
    lm_ref = float(F.mse_loss(X_fake.double(), X.double()))
    assert abs(float(lm.detach()) - lm_ref) <= 1e-5 * lm_ref
    assert float(miou_m) == float(miou)
    gim, gam = torch.autograd.grad(lm * gup, [i3, a3])
    i4, a4 = image.clone().requires_grad_(True), alpha.clone().requires_grad_(True)
    rim, ram = torch.autograd.grad(F.mse_loss(torch.cat((i4, a4), dim=3).permute(0, 3, 1, 2), X) * gup, [i4, a4])
    assert float((gim - rim).abs().max()) < 1e-9 and float((gam - ram).abs().max()) < 1e-9


# ------------------------------------------------------------------------------------------------ eval-mode network
def test_reconstruction_network_eval_mode_matches_reference_golden():
    from models import reconstruction
    d = np.load(os.path.join(GOLDEN, "recon_eval_reference.npz"))
    net = RE.set_running_stats(RC.build(reconstruction)).cuda().eval()
    x, _, _ = RC.inputs()
    with torch.no_grad():
        tex, mesh_map = net(x.cuda())
    assert tex.shape == (8, 3, 128, 128) and mesh_map.shape == (8, 3, 32, 32)

    def close(a, ref, tol):
        err = float(np.abs(a.cpu().numpy() - ref).max())
        assert err <= tol * max(float(np.abs(ref).max()), 1e-6), (err, tol)
    close(tex[:, :, ::8, ::8], d["evalnet.tex_probe"], 5e-2)
    assert abs(float(tex.double().sum()) - float(d["evalnet.tex_sum"])) < 2e-2 * tex.numel() ** 0.5 * 5
    close(mesh_map, d["evalnet.mesh_map"], 2e-2)
    for t in (tex, mesh_map):                               # symmetric output: mirrored about the seam at a quarter width
        qw = t.shape[3] // 4
        assert torch.equal(t[..., :qw], t[..., qw:2 * qw].flip(3)) and torch.equal(t[..., 3 * qw:], t[..., 2 * qw:3 * qw].flip(3))


# ------------------------------------------------------------------------------------------------ validation pass
def eval_trainer(tpl, loss):
    from reconstruction_training import ReconTrainer, default_args
    torch.manual_seed(4321)
    tr = ReconTrainer(default_args(optimize_z0=True, loss=loss), tpl, dataset_size=4722, device=DEV)
    RE.set_running_stats(tr.generator)
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():                                   # a mesh head with a signal, so the flat loss sees a deformation
        tr.generator.conv_mesh.weight.copy_(torch.randn(tr.generator.conv_mesh.weight.shape, generator=g) * 0.02)
    RE.perturb_dataset_params(tr.dataset_params)
    return tr


@pytest.mark.parametrize("loss", RE.CRITERIA)
def test_evaluate_equals_hand_composition(tpl31, loss):
    tr = eval_trainer(tpl31, loss)
    batches = [disk_batch(4, 20), disk_batch(4, 21)]
    seen = []
    h = tr.generator.register_forward_hook(lambda m, i, o: seen.append(tuple(t.clone() for t in o)))
    try:
        got = tr.evaluate(batches)
    finally:
        h.remove()
    crit = torch_criterion(loss)
    tot, n = np.zeros(3), 0
    with torch.no_grad():
        t_mean, s_mean = tr.dataset_params(None, 'deltas')
        z0_mean = tr.dataset_params(None, 'z0')
        for (X, s, t, q, _), (pred_tex, mesh_map) in zip(batches, seen):
            B = X.shape[0]
            own_tex, own_mesh = tr.generator(X)             # the pass used this network, in eval mode
            assert float((own_tex - pred_tex).abs().max()) < 1e-5 and float((own_mesh - mesh_map).abs().max()) < 1e-5
            raw, vtx = tpl31.vertices_and_pose(mesh_map, s + s_mean, t + t_mean, q, z0_mean.expand(B, 1).contiguous())
            image, alpha = tpl31.forward_renderer(tr.renderer, vtx, pred_tex)
            recon, miou = crit(image, alpha, X)
            flat = OM.loss_flat(tpl31.mesh.ff, tpl31.mesh.faces.shape[0], tpl31.compute_normals(raw))
            tot += B * np.array([recon.item(), flat.item(), miou.item()])
            n += B
    assert got["N"] == n == 8
    for k, want in zip(("recon_loss", "flat_loss"), tot / n):
        assert abs(got[k] - want) <= 1e-5 * abs(want), (k, got[k], want)
    assert got["miou"] == tot[2] / n
    assert 0 < got["miou"] < 1 and got["flat_loss"] > 0


def test_evaluate_has_no_batch_coupling(tpl31):
    """Eval-mode batch norm couples no samples (training mode would move these values by ~1e-1).  What does depend on
    the batch size is the fp32 GEMM algorithm torch picks for the three nn.Linear layers: the encoder output differs by
    ~1e-7, the decoder carries that to ~1e-4 of the displacement map, and the flat loss of this strongly deformed mesh
    (~300) moves by ~6e-5 relative on an H100 — hence its looser limit."""
    tr = eval_trainer(tpl31, "mse")
    X, s, t, q, idx = disk_batch(8, 30)
    one = tr.evaluate([(X, s, t, q, idx)])
    two = tr.evaluate([(X[:4], s[:4], t[:4], q[:4], idx[:4]), (X[4:], s[4:], t[4:], q[4:], idx[4:])])
    assert one["N"] == two["N"] == 8
    for k, rel in (("recon_loss", 1e-5), ("miou", 1e-5), ("flat_loss", 3e-4)):
        assert abs(one[k] - two[k]) <= rel * abs(one[k]), (k, one[k], two[k])


# ------------------------------------------------------------------------------------------------ L1 training step
def test_l1_training_step_matches_torch_loss(tpl31, monkeypatch):
    import reconstruction_training as RT
    from reconstruction_training import ReconTrainer, default_args
    X, s, t, q, idx = disk_batch(8, 40)
    out = []
    for use_torch in (False, True):
        if use_torch:
            monkeypatch.setattr(RT, "rgba_l1_iou", torch_criterion("l1"))
        torch.manual_seed(4321)
        tr = ReconTrainer(default_args(loss='l1'), tpl31, dataset_size=4722, device=DEV)
        loss, recon, flat, miou = tr.step(X, s, t, q, idx)
        out.append((float(loss), float(recon), float(miou),
                    {n: float(p.grad.norm()) for n, p in tr.generator.named_parameters() if p.grad is not None}))
    (l_k, r_k, m_k, g_k), (l_t, r_t, m_t, g_t) = out
    assert abs(l_k - l_t) <= 1e-5 * abs(l_t) and abs(r_k - r_t) <= 1e-5 * abs(r_t) and abs(m_k - m_t) < 1e-4
    assert g_k.keys() == g_t.keys() and len(g_k) > 10
    # the step itself is not bit-reproducible (atomic accumulation in the backward): the SAME step run twice on an H100
    # moves the gradient norms of the encoder's batch-norm affine parameters (~1e-2 of the largest norm) by up to
    # 1.2e-4 relative — hence the floor of 1e-5 of the largest norm beside the 1e-4 relative limit
    floor = 1e-5 * max(g_t.values())
    for n in g_t:
        assert abs(g_k[n] - g_t[n]) <= 1e-4 * g_t[n] + floor, (n, g_k[n], g_t[n])


# ------------------------------------------------------------------------------------------------ turntable
def test_render_multiview_equals_direct_renders(tpl31):
    from rendering.utils import qmul, qrot
    tr = eval_trainer(tpl31, "mse")
    X, *_ = disk_batch(3, 50)
    idx = 2
    with torch.no_grad():
        tr.generator.eval()
        pred_tex, mesh_map = tr.generator(X)
        raw = tpl31.vertices_and_pose(mesh_map)[0]
    tile = tr.render_multiview(raw, pred_tex, idx)
    assert tile.shape == (2 * R, 4 * R, 3) and tile.dtype == np.float32

    def about(axis, deg, factor=1.0):                       # the reference's turntable quaternions (:192-203)
        rad = deg / 180 * np.pi * factor
        v = [np.cos(-rad / 2), 0, 0, 0]
        v[axis] = np.sin(-rad / 2)
        return torch.Tensor(v).to(DEV)
    q0 = qmul(about(3, -90), about(2, 110))
    for k, angle in enumerate((0, 45, 90, 135, 180, 225, 270, 315)):
        rot = qmul(q0, about(3, angle, 0.8))[None]
        with torch.no_grad():
            vtx = qrot(rot, raw[idx:idx + 1]) * 0.9
            vtx[:, :, 1:] *= -1
            view, _ = tpl31.forward_renderer(tr.renderer, vtx, pred_tex[idx:idx + 1].contiguous())
        want = (view[0].cpu().numpy() + 1) / 2
        r, c = divmod(k, 4)
        got = tile[r * R:(r + 1) * R, c * R:(c + 1) * R]
        assert np.abs(got - want).max() <= 1e-6, k
    assert tile.min() >= 0 and tile.max() <= 1 and tile.std() > 0.01
