"""Host-side logic of the reconstruction validation pass, turntable render and L1 criterion (CPU), against
tests/golden/recon_eval_reference.npz: the reference's evaluate_all / render_multiview / training loop EXECUTED from
run_reconstruction.py's syntax tree on recon_step_common's stand-ins (make_golden_recon_eval.py).  ReconTrainer runs on
the same stand-ins with its fused CUDA pieces (RGBA loss + IoU kernel, flat-loss kernel, fused vertex pipeline)
replaced by their torch definitions.  Also: the eval-mode wiring of models.reconstruction, and the new C-ABI exports'
argument checks."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import recon_common as RC           # noqa: E402
import recon_eval_common as RE      # noqa: E402
import recon_step_common as RS      # noqa: E402


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "recon_eval_reference.npz"))


def torch_criteria(monkeypatch):
    """b3d.mesh.rgba_{mse,l1}_iou and utils.losses.loss_flat as their torch definitions (run_reconstruction.py:429-436)."""
    import reconstruction_training as RT
    from oracle import mesh as OM

    def fused(loss):
        def fn(image, alpha, X_real):
            X_fake = torch.cat((image, alpha), dim=3).permute(0, 3, 1, 2)
            return loss(X_fake, X_real), OM.mean_iou(X_fake[:, 3], X_real[:, 3])
        return fn
    monkeypatch.setattr(RT, "rgba_mse_iou", fused(F.mse_loss))
    monkeypatch.setattr(RT, "rgba_l1_iou", fused(F.l1_loss))
    monkeypatch.setattr(RT, "loss_flat", lambda mesh, norms: OM.loss_flat(mesh.ff, mesh.faces.shape[0], norms))
    return RT


def standin_trainer(RT, args, generator):
    """ReconTrainer wired to the stand-ins (its constructor builds the CUDA network)."""
    from models.reconstruction import DatasetParams
    from oracle import mesh as OM
    tpl = RS.Template()
    tpl.vertices_and_pose = lambda m, s, t, r, z=None: (lambda raw: (raw, OM.transform_vertices(raw, s, t, r, z)))(tpl.get_vertex_positions(m))
    tr = object.__new__(RT.ReconTrainer)
    tr.args, tr.tpl, tr.world, tr.renderer = args, tpl, 1, None
    tr.generator = generator
    tr.optimizer = torch.optim.Adam(tr.generator.parameters(), lr=args.lr)
    tr.dataset_params = DatasetParams(args, 10)
    tr.optimizer_dataset = torch.optim.Adam(tr.dataset_params.parameters(), lr=args.lr_dataset)
    tr.flat_warmup = torch.full((), 10.0)
    return tr


def eval_trainer(RT, deltas, z0, loss):
    args = RS.make_args(deltas, z0)
    args.loss = loss
    tr = standin_trainer(RT, args, RE.set_running_stats(RS.build_net()))
    RE.perturb_dataset_params(tr.dataset_params)
    return tr


def log_line(r):
    return '[TEST] recon_loss {:.5f}, flat_loss {:.5f}, mIoU {:.5f}, N {}'.format(r["recon_loss"], r["flat_loss"], r["miou"], r["N"])


@pytest.mark.parametrize("loss", RE.CRITERIA)
@pytest.mark.parametrize("tag,deltas,z0", RE.POSES)
def test_evaluate_matches_the_reference_validation_pass(loss, tag, deltas, z0, gold, monkeypatch):
    RT = torch_criteria(monkeypatch)
    tr = eval_trainer(RT, deltas, z0, loss)
    tr.generator.train()
    r = tr.evaluate(RE.eval_batches())
    assert not tr.generator.training
    assert log_line(r) == str(gold[f"eval.{loss}.{tag}.log"])
    ref = gold[f"eval.{loss}.{tag}.totals"]
    got = np.array([r["recon_loss"], r["flat_loss"], r["miou"], r["N"]])
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=0)
    assert isinstance(r["N"], int) and all(isinstance(r[k], float) for k in ("recon_loss", "flat_loss", "miou"))


def test_evaluate_keeps_the_nan_iou_of_an_empty_batch(monkeypatch):
    """Predicted and target alpha both empty: intersection / union = 0 / 0, a NaN mIoU exactly as the reference logs."""
    RT = torch_criteria(monkeypatch)
    tr = eval_trainer(RT, True, False, "mse")
    tr.tpl.forward_renderer = lambda renderer, vtx, tex: (torch.zeros(vtx.shape[0], RS.H, RS.H, 3), torch.zeros(vtx.shape[0], RS.H, RS.H, 1))
    X, s, t, r, idx = RE.eval_batches()[0]
    X = X.clone()
    X[:, 3] = 0
    out = tr.evaluate([(X, s, t, r, idx)])
    assert np.isnan(out["miou"]) and np.isfinite(out["recon_loss"]) and out["N"] == 4


def test_render_multiview_matches_the_reference(gold, monkeypatch):
    RT = torch_criteria(monkeypatch)
    tr = standin_trainer(RT, RS.make_args(), RS.build_net())
    tile = tr.render_multiview(torch.tensor(gold["multiview.raw_vtx"]), torch.tensor(gold["multiview.pred_tex"]), RE.MULTIVIEW_IDX)
    ref = gold["multiview.tile"]
    assert tile.shape == ref.shape == (2 * RS.H, 4 * RS.H, 3) and tile.dtype == ref.dtype
    assert np.abs(tile - ref).max() <= 1e-6


@pytest.mark.parametrize("tag,deltas,z0", RE.POSES)
def test_l1_training_iteration_matches_the_reference_loop(tag, deltas, z0, gold, monkeypatch):
    """Tolerances of test_recon_hostlogic.py::test_training_iteration_matches_the_reference_loop."""
    RT = torch_criteria(monkeypatch)
    args = RS.make_args(deltas, z0)
    args.loss = "l1"
    tr = standin_trainer(RT, args, RS.build_net())
    losses = []
    for i, (X, s, t, r, idx) in enumerate(RS.batches()):
        loss, recon, flat, miou = tr.step(X, s, t, r, idx.squeeze(-1))
        losses.append(float(loss))
        if i == 0:
            ref = str(gold[f"l1step.{tag}.log0"])
            assert f"recon_loss {float(recon):.5f} flat_loss {float(flat):.5f} total {float(loss):.5f} iou {float(miou):.5f}" in ref
    assert np.abs(np.array(losses) - gold[f"l1step.{tag}.g_curve"]).max() < 2e-6
    assert abs(float(tr.flat_warmup) - float(gold[f"l1step.{tag}.flat_warmup"])) < 1e-5
    for k, v in tr.generator.state_dict().items():
        assert np.abs(v.numpy().astype(np.float64) - gold[f"l1step.{tag}.net.{k}"]).max() < 1e-4, k
    for k, v in tr.dataset_params.state_dict().items():
        assert np.abs(v.numpy() - gold[f"l1step.{tag}.dp.{k}"]).max() < 1e-4, k


def test_l1_path_calls_the_l1_kernel_wrapper(monkeypatch):
    """loss='l1' goes through reconstruction_training.rgba_l1_iou, 'mse' through rgba_mse_iou."""
    RT = torch_criteria(monkeypatch)
    called = []
    for name in ("rgba_mse_iou", "rgba_l1_iou"):
        fn = getattr(RT, name)
        monkeypatch.setattr(RT, name, lambda *a, _fn=fn, _n=name: called.append(_n) or _fn(*a))
    for loss in ("mse", "l1"):
        args = RS.make_args()
        args.loss = loss
        X, s, t, r, idx = RS.batches()[0]
        standin_trainer(RT, args, RS.build_net()).step(X, s, t, r, idx.squeeze(-1))
    assert called == ["rgba_mse_iou", "rgba_l1_iou"]


@pytest.mark.parametrize("loss", ["huber", "MSE", ""])
def test_unknown_criterion_is_rejected(loss):
    import reconstruction_training as RT
    with pytest.raises(ValueError, match="loss="):
        RT.ReconTrainer(RT.default_args(loss=loss), None, 10, device="cpu")


def test_l1_exports_reject_bad_arguments_without_gpu():
    import b3d
    lib = b3d.lib
    assert lib.b3d_rgba_l1_iou_fwd(None, None, None, 1, 4, 4, None, None, None) == -1
    assert b"b3d_rgba_l1_iou_fwd: bad arguments" in lib.b3d_last_error()
    assert lib.b3d_rgba_l1_bwd(None, None, None, 0, 4, 4, None, None, None, None) == -1
    assert b"b3d_rgba_l1_bwd: bad arguments" in lib.b3d_last_error()


def test_eval_mode_wiring_matches_reference_golden_on_cpu(gold, monkeypatch):
    """models.reconstruction in eval mode (running statistics from recon_eval_common) with TCConv2d -> nn.Conv2d.forward
    and pad_x -> F.pad / wrap-around cat reproduces the reference's eval-mode forward to fp32 round-off."""
    from models import gan, reconstruction

    def pad_x_cpu(t, amount, mode):
        if mode == reconstruction.REPLICATE:
            return F.pad(t, (amount, amount, 0, 0), mode='replicate')
        return torch.cat((t[..., -amount:], t, t[..., :amount]), dim=3)

    monkeypatch.setattr(gan.TCConv2d, "forward", lambda self, x, **kw: nn.Conv2d.forward(self, x))
    monkeypatch.setattr(reconstruction, "pad_x", pad_x_cpu)
    torch.set_num_threads(8)
    net = RE.set_running_stats(RC.build(reconstruction)).eval()
    x, _, _ = RC.inputs()
    with torch.no_grad():
        tex, mesh_map = net(x)
    assert np.abs(tex[:, :, ::8, ::8].numpy() - gold["evalnet.tex_probe"]).max() < 2e-4
    assert np.abs(mesh_map.numpy() - gold["evalnet.mesh_map"]).max() < 1e-4
    assert abs(float(tex.double().sum()) - float(gold["evalnet.tex_sum"])) < 1e-2
