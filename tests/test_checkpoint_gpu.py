"""Checkpoints of the CUDA trainers on the H100:
  * save -> fresh trainer -> resume restores every parameter, buffer (spectral-norm u / v, BN running statistics,
    num_batches_tracked) and Adam tensor bit for bit, with `step` on the device for the fused / capturable Adams, and the
    counters, curves and flat-loss warm-up factor (GAN at 256², nd 2; reconstruction with deltas + z0; capturable or not);
  * an interrupted run (epoch 0, save, load into a fresh trainer, epoch 1) equals an uninterrupted one within 4x the
    run-to-run difference measured in the same test (the split-K weight-gradient atomics make two identical runs differ
    by rounding, DESIGN §4 "Determinism");
  * an 'evaluate'-mode load feeds the evaluations: the running-average generator renders bit-identical textures and the
    FID features agree, and ReconTrainer.evaluate gives the original trainer's values."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, ROOT

sys.path.insert(0, GOLDEN)
sys.path.insert(0, ROOT)
import gan_common as GC          # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def tpl16():
    from rendering.mesh_template import MeshTemplate
    from tools.uvsphere import write_uvsphere_obj
    return MeshTemplate(write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_16rings.obj"), rings=16), device=DEV)


@pytest.fixture(scope="module")
def tpl31():
    from rendering.mesh_template import MeshTemplate
    from tools.uvsphere import write_uvsphere_obj
    return MeshTemplate(write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), "uvsphere_31rings.obj"), rings=31), device=DEV)


def gan_trainer(tpl, seed, capturable=False, **kw):
    import bench
    from gan_training import GANTrainer
    args = bench.gan_args(256, 2)
    for k, v in kw.items():
        setattr(args, k, v)
    torch.manual_seed(seed)
    return GANTrainer(args, mesh_template=tpl, device=DEV, capturable=capturable)


def gan_batches(n, seed, B=2):
    args = GC.make_args(256, 2)
    out = []
    for i in range(n):
        z, c, alpha, tex, mesh = GC.inputs(args, B=B, seed=seed + i)
        out.append(dict(X_tex=tex.to(DEV), X_alpha=alpha.to(DEV), X_mesh=mesh.to(DEV), C=c.to(DEV), noise=z.to(DEV)))
    return out


def recon_trainer(tpl, seed, capturable=False):
    from reconstruction_training import ReconTrainer, default_args
    torch.manual_seed(seed)
    return ReconTrainer(default_args(optimize_z0=True), tpl, dataset_size=20, device=DEV, capturable=capturable)


def recon_batches(n, seed, B=2, R=256):
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, R), torch.linspace(-1, 1, R), indexing="ij")
    disk = ((yy * yy + xx * xx) < 0.45).float()
    out = []
    for _ in range(n):
        X = torch.rand(B, 4, R, R, generator=g) * 2 - 1
        X[:, 3] = disk
        X[:, :3] *= disk
        b = (X, 0.55 + 0.3 * torch.rand(B, 1, generator=g), (torch.rand(B, 3, generator=g) - 0.5) * 0.3,
             F.normalize(torch.randn(B, 4, generator=g), dim=-1), torch.randint(0, 40, (B,), generator=g))
        out.append(tuple(v.to(DEV) for v in b))
    return out


def gan_state(tr):
    t = tr.trainer
    mods = (("g", t.generator), ("avg", t.generator_running_avg), ("d", t.discriminator))
    return state(mods, (("opt_g", tr.optimizer_g), ("opt_d", tr.optimizer_d)))


def recon_state(tr):
    return state((("net", tr.generator), ("dp", tr.dataset_params)), (("opt", tr.optimizer), ("opt_dp", tr.optimizer_dataset)))


def state(mods, opts):
    out = {}
    for name, m in mods:
        out.update({f"{name}.{k}": v.detach().clone() for k, v in m.state_dict().items()})
    for name, opt in opts:
        for i, p in enumerate(q for g in opt.param_groups for q in g["params"]):
            for k, v in opt.state[p].items():
                out[f"{name}.{i}.{k}"] = v.detach().clone()
    return out


def assert_identical(a, b):
    assert set(a) == set(b)
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].device == b[k].device and torch.equal(a[k], b[k]), k


# ------------------------------------------------------------------------------------------------ round trip
@pytest.mark.parametrize("capturable", [False, True])
def test_gan_round_trip_is_exact(tpl16, capturable, tmp_path):
    tr = gan_trainer(tpl16, 1, capturable)
    tr.train_epoch(gan_batches(4, 10))                 # G D D G
    saved = gan_state(tr)
    assert any("weight_u" in k for k in saved) and any("running_mean" in k for k in saved)
    assert any("num_batches_tracked" in k for k in saved) and all(saved[k].is_cuda for k in saved if k.endswith(".step"))
    tr.save_checkpoint(str(tmp_path / "c.pth"))
    fresh = gan_trainer(tpl16, 2, capturable)
    fresh.load_checkpoint(str(tmp_path / "c.pth"), "resume")
    assert_identical(gan_state(fresh), saved)
    assert (fresh.epoch, fresh.total_it) == (tr.epoch, tr.total_it) == (1, 4)
    for k in ("g_curve", "d_fake_curve", "d_real_curve", "flat_curve"):
        assert getattr(fresh, k) == getattr(tr, k)
    assert len(tr.g_curve) == 3 and len(tr.d_fake_curve) == 3 and len(tr.flat_curve) == 3
    assert fresh.optimizer_g.param_groups[0]["fused"] and fresh.optimizer_g.param_groups[0]["capturable"] == capturable


@pytest.mark.parametrize("capturable", [False, True])
def test_recon_round_trip_is_exact(tpl31, capturable, tmp_path):
    tr = recon_trainer(tpl31, 1, capturable)
    tr.train_epoch(recon_batches(3, 5))
    saved = recon_state(tr)
    assert {"dp.ds_translation", "dp.ds_z0"} <= set(saved) and any("running_var" in k for k in saved)
    tr.save_checkpoint(str(tmp_path / "c.pth"))
    fresh = recon_trainer(tpl31, 2, capturable)
    fresh.load_checkpoint(str(tmp_path / "c.pth"), "resume")
    assert_identical(recon_state(fresh), saved)
    assert torch.equal(fresh.flat_warmup, tr.flat_warmup) and abs(float(tr.flat_warmup) - 9.7) < 1e-5
    assert (fresh.epoch, fresh.total_it) == (tr.epoch, tr.total_it) == (1, 3)


# ------------------------------------------------------------------------------------------------ resume == no interruption
def test_gan_resume_equals_an_uninterrupted_run(tpl16, tmp_path):
    """Two epochs of 4 iterations; lr_decay_after = 0 and epochs = 4 make the decay fire at the boundary (factor 0.75)."""
    sched = dict(lr_decay_after=0, epochs=4)
    e0, e1 = gan_batches(4, 20), gan_batches(4, 30)

    def uninterrupted():
        tr = gan_trainer(tpl16, 7, **sched)
        losses = [float(x) for x in tr.train_epoch(e0) + tr.train_epoch(e1)]
        return tr, losses
    u1, l1 = uninterrupted()
    u2, l2 = uninterrupted()
    first = gan_trainer(tpl16, 7, **sched)
    li = [float(x) for x in first.train_epoch(e0)]
    first.save_checkpoint(str(tmp_path / "c.pth"))
    second = gan_trainer(tpl16, 8, **sched)
    second.load_checkpoint(str(tmp_path / "c.pth"), "resume")
    assert second.optimizer_g.param_groups[0]["lr"] == 0.75 * 1e-4 and second.optimizer_d.param_groups[0]["lr"] == 0.75 * 4e-4
    li += [float(x) for x in second.train_epoch(e1)]
    assert (second.epoch, second.total_it) == (u1.epoch, u1.total_it) == (2, 8)
    assert second.g_curve[:len(first.g_curve)] == first.g_curve and len(second.g_curve) == len(u1.g_curve)
    s1, s2, si = gan_state(u1), gan_state(u2), gan_state(second)
    noise = max(float((s2[k].double() - s1[k].double()).abs().max()) for k in s1)
    dev = max(float((si[k].double() - s1[k].double()).abs().max()) for k in s1)
    lnoise = max(abs(a - b) for a, b in zip(l1, l2))
    ldev = max(abs(a - b) for a, b in zip(l1, li))
    print(f"state: resumed vs uninterrupted {dev:.3e}, run-to-run {noise:.3e}; losses {ldev:.3e} vs {lnoise:.3e}")
    assert dev <= 4 * noise + 1e-7 and ldev <= 4 * lnoise + 1e-7


# ------------------------------------------------------------------------------------------------ evaluate mode
def test_evaluate_mode_load_feeds_the_fid_evaluation(tpl16, tmp_path):
    from fid_common import randomize_inception
    from fid_evaluation import FIDEvaluator
    from utils.inception import InceptionV3
    tr = gan_trainer(tpl16, 3)
    tr.train_epoch(gan_batches(4, 40))
    tr.save_checkpoint(str(tmp_path / "c.pth"))
    ev_tr = gan_trainer(tpl16, 4)
    ev_tr.load_checkpoint(str(tmp_path / "c.pth"), "evaluate")
    a, b = tr.trainer.generator_running_avg.eval(), ev_tr.trainer.generator_running_avg.eval()
    z, c, *_ = GC.inputs(GC.make_args(256, 2), B=3, seed=77)
    with torch.no_grad():
        ta, ma, _ = a(z.to(DEV), c.to(DEV), None, return_attention=True)
        tb, mb, _ = b(z.to(DEV), c.to(DEV), None, return_attention=True)
    assert torch.equal(ta, tb) and torch.equal(ma, mb)
    inc = randomize_inception(InceptionV3([2], weights=None), 6)
    g = torch.Generator().manual_seed(5)
    data = [{"idx": torch.arange(3), "class": torch.randint(0, 200, (3, 1), generator=g),
             "rotation": F.normalize(torch.randn(3, 4, generator=g), dim=-1), "scale": 0.5 + 0.3 * torch.rand(3, generator=g),
             "translation": (torch.rand(3, 3, generator=g) - 0.5) * 0.2, "image": torch.rand(3, 3, 299, 299, generator=g)}
            for _ in range(2)]
    fa = FIDEvaluator(a, tpl16, inception=inc, device=DEV).evaluate(data, seed=1234, keep_features=True)
    fb = FIDEvaluator(b, tpl16, inception=inc, device=DEV).evaluate(data, seed=1234, keep_features=True)
    xa, xb = fa["features"]["combined"], fb["features"]["combined"]
    assert float((xa - xb).abs().max()) <= 1e-5 * float(xa.abs().max())
    assert abs(fa["fid"] - fb["fid"]) <= 1e-4 * abs(fa["fid"])


def test_evaluate_mode_load_feeds_the_validation_pass(tpl31, tmp_path):
    tr = recon_trainer(tpl31, 1)
    tr.train_epoch(recon_batches(3, 5))
    tr.save_checkpoint(str(tmp_path / "c.pth"))
    ev_tr = recon_trainer(tpl31, 2)
    ev_tr.load_checkpoint(str(tmp_path / "c.pth"), "evaluate")
    val = recon_batches(2, 9, B=3)
    ra, rb = tr.evaluate(val), ev_tr.evaluate(val)
    assert ra["N"] == rb["N"] == 6
    for k in ("recon_loss", "flat_loss", "miou"):
        assert abs(ra[k] - rb[k]) <= 1e-6 * abs(ra[k]), (k, ra[k], rb[k])
    assert not ev_tr.optimizer.state and float(ev_tr.flat_warmup) == 10.0
