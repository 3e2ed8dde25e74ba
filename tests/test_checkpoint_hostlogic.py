"""Checkpoints, resume, epoch schedules and the best-epoch search of GANTrainer / ReconTrainer against the reference's own
epoch layer (CPU).  tests/golden/make_golden_checkpoint.py executed main.py's and run_reconstruction.py's training loops,
loading blocks and save_checkpoint closures on the stand-ins of wrapper_common.py / recon_step_common.py: it stored the
checkpoints the reference wrote (as data, saved back to files here by `ref_files`) and how the reference continues from them
in checkpoint_reference.npz.  Here
the trainers run on the same stand-ins (their fused CUDA pieces replaced by the torch definitions, as in
test_gan_hostlogic.py / test_recon_hostlogic.py)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import GOLDEN, PKG, ROOT

sys.path.insert(0, GOLDEN)
import checkpoint_common as CC     # noqa: E402
import recon_step_common as RS     # noqa: E402
import wrapper_common as WC        # noqa: E402

TOL = 2e-6


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "checkpoint_reference.npz"))


@pytest.fixture(scope="module")
def ref_files(golden, tmp_path_factory):
    """The reference-written checkpoints, saved back to files: {'gan_ckpt' | 'gan_ckpt_numstep' | 'recon_ckpt': path}."""
    d = tmp_path_factory.mktemp("reference_checkpoints")
    out = {}
    for name in ("gan_ckpt", "gan_ckpt_numstep", "recon_ckpt"):
        out[name] = str(d / f"{name}.pth")
        torch.save(CC.decode(golden, name), out[name])
    return out


def torch_pieces(monkeypatch):
    """Replace the fused CUDA losses of both trainers by their torch definitions."""
    import gan_training as GT
    import reconstruction_training as RT
    from oracle import mesh as OM

    def rgba_mse_iou(image, alpha, X_real):
        X_fake = torch.cat((image, alpha), dim=3).permute(0, 3, 1, 2)
        return torch.nn.functional.mse_loss(X_fake, X_real), OM.mean_iou(X_fake[:, 3], X_real[:, 3])
    flat = lambda mesh, norms: OM.loss_flat(mesh.ff, mesh.faces.shape[0], norms)
    monkeypatch.setattr(GT, "loss_flat", flat)
    monkeypatch.setattr(RT, "loss_flat", flat)
    monkeypatch.setattr(RT, "rgba_mse_iou", rgba_mse_iou)
    return GT, RT


def gan_trainer(GT, args, seed, fused=False):
    """A GANTrainer on the stand-in networks (the constructor builds the CUDA networks; wire the stand-ins instead)."""
    gi, D = WC.build(seed)
    tr = object.__new__(GT.GANTrainer)
    tr.args, tr.mesh_template, tr.world, tr.total_it, tr.epoch = args, RS.Template(map_size=8), 1, 0, 0
    tr.g_curve, tr.d_fake_curve, tr.d_real_curve, tr.flat_curve = [0], [0], [0], [0]
    tr.trainer = GT.ModelWrapper(args, gi, D).train()
    tr.optimizer_g = torch.optim.Adam(tr.trainer.generator.parameters(), lr=args.lr_g, betas=(0.0, 0.9), fused=fused)
    tr.optimizer_d = torch.optim.Adam(tr.trainer.discriminator.parameters(), lr=args.lr_d, betas=(0.0, 0.9), fused=fused)
    return tr


def recon_trainer(RT, args, seed, fused=False, dataset_params=True):
    from models.reconstruction import DatasetParams
    from oracle import mesh as OM
    tpl = RS.Template()
    tpl.vertices_and_pose = lambda m, s, t, r, z=None: (lambda raw: (raw, OM.transform_vertices(raw, s, t, r, z)))(tpl.get_vertex_positions(m))
    tr = object.__new__(RT.ReconTrainer)
    tr.args, tr.tpl, tr.world, tr.renderer, tr.epoch, tr.total_it = args, tpl, 1, None, 0, 0
    tr.generator = RS.build_net(seed)
    tr.optimizer = torch.optim.Adam(tr.generator.parameters(), lr=args.lr, fused=fused)
    tr.dataset_params = tr.optimizer_dataset = None
    if dataset_params:
        tr.dataset_params = DatasetParams(args, 10)
        tr.optimizer_dataset = torch.optim.Adam(tr.dataset_params.parameters(), lr=args.lr_dataset, fused=fused)
    tr.flat_warmup = torch.full((), 10.0)
    return tr


def gan_args_b():
    a = CC.gan_args()
    a.epochs, a.lr_decay_after = CC.GAN_EPOCHS_B, CC.GAN_DECAY_AFTER_B
    return a


def recon_args_b():
    a = CC.recon_args()
    a.epochs, a.lr_decay_every = CC.RECON_EPOCHS_B, CC.RECON_DECAY_EVERY
    return a


def close(got, ref, tol, what):
    got = got.detach().double().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = np.abs(got - ref).max() if got.size else 0.0
    assert err <= tol, (what, err)


def check_states(golden, prefix, mods, opts, tol):
    for name, mod in mods:
        for k, v in mod.state_dict().items():
            close(v, golden[f"{prefix}.{name}.{k}"], tol, (name, k))
    for name, opt in opts:
        st = CC.adam_state(opt)
        assert {f"{prefix}.{name}.{k}" for k in st} == {k for k in golden.files if k.startswith(f"{prefix}.{name}.")}
        for k, v in st.items():
            close(v, golden[f"{prefix}.{name}.{k}"], tol, (name, k))


def layout(x):
    """A structural fingerprint: key sets and nesting, Python types, tensor shapes and dtypes (not values or devices)."""
    if isinstance(x, torch.Tensor):
        return ("tensor", tuple(x.shape), str(x.dtype))
    if isinstance(x, dict):
        return ("dict", {k: layout(v) for k, v in x.items()})
    if isinstance(x, (list, tuple)):
        return (type(x).__name__, [layout(v) for v in x])
    return type(x).__name__


# ------------------------------------------------------------------------------------------------ format
@pytest.mark.parametrize("fused", [False, True])
def test_gan_checkpoint_has_the_reference_layout(fused, golden, tmp_path, monkeypatch):
    """A checkpoint written by GANTrainer has the reference file's keys, nesting, Python types, tensor shapes / dtypes and
    optimiser param_groups / state layout, whichever Adam implementation ran (the flags are written as a plain Adam's)."""
    GT, _ = torch_pieces(monkeypatch)
    ref = CC.decode(golden, "gan_ckpt")
    tr = gan_trainer(GT, CC.gan_args(), CC.GAN_SEED_A, fused=fused)
    torch.manual_seed(CC.GAN_NOISE_A)
    for _ in range(CC.GAN_EPOCHS_A):
        tr.train_epoch(CC.gan_inputs())
    tr.save_checkpoint(str(tmp_path / "c.pth"))
    mine = torch.load(str(tmp_path / "c.pth"))
    ref_args, mine_args = ref.pop("args"), mine.pop("args")
    assert isinstance(mine_args, dict) and isinstance(ref_args, dict) and set(vars(CC.gan_args())) <= set(mine_args)
    assert layout(mine) == layout(ref)
    for k in ("optimizer_g", "optimizer_d"):
        assert mine[k]["param_groups"] == ref[k]["param_groups"]
    assert mine["epoch"] == ref["epoch"] and mine["iteration"] == ref["iteration"]
    for k in ("g_curve", "d_fake_curve", "d_real_curve", "flat_curve"):
        assert mine[k][0] == 0 and type(mine[k][0]) is int
        close(mine[k], np.array(ref[k], dtype=np.float64), TOL, k)


def test_recon_checkpoint_has_the_reference_layout_plus_flat_warmup(golden, tmp_path, monkeypatch):
    _, RT = torch_pieces(monkeypatch)
    ref = CC.decode(golden, "recon_ckpt")
    a = CC.recon_args()
    a.lr_decay_every = CC.RECON_DECAY_EVERY
    tr = recon_trainer(RT, a, CC.RECON_SEED_A, fused=True)
    for _ in range(CC.RECON_EPOCHS_A):
        tr.train_epoch(CC.recon_batches())
    tr.save_checkpoint(str(tmp_path / "c.pth"))
    mine = torch.load(str(tmp_path / "c.pth"))
    assert isinstance(mine.pop("args"), dict) and isinstance(ref.pop("args"), dict)
    assert isinstance(mine.pop("flat_warmup"), float) and "flat_warmup" not in ref
    assert layout(mine) == layout(ref)
    for k in ("optimizer", "optimizer_dataset_params"):
        assert mine[k]["param_groups"] == ref[k]["param_groups"]        # incl. the halved network rate at epoch 2
    assert mine["epoch"] == ref["epoch"] == 2 and mine["iteration"] == ref["iteration"] == 8
    tr = recon_trainer(RT, a, CC.RECON_SEED_A, dataset_params=False)
    tr.save_checkpoint(str(tmp_path / "n.pth"))
    mine = torch.load(str(tmp_path / "n.pth"))
    assert mine["dataset_params"] is None and mine["optimizer_dataset_params"] is None


# ------------------------------------------------------------------------------------------------ reference file -> our trainer
@pytest.mark.parametrize("name,fused", [("gan_ckpt", False), ("gan_ckpt_numstep", False), ("gan_ckpt", True)],
                         ids=["tensor-step", "numeric-step", "fused"])
def test_gan_resume_from_reference_checkpoint_continues_the_reference_run(name, fused, golden, ref_files, monkeypatch):
    """--continue_train from the reference's checkpoint_2.pth, then four epochs (the G / D phase continues mid-cycle, the
    linear decay starts at epoch 3): curves, learning rates per epoch, iteration counter, networks and Adam state."""
    GT, _ = torch_pieces(monkeypatch)
    tr = gan_trainer(GT, gan_args_b(), CC.GAN_SEED_B, fused=fused)
    tr.load_checkpoint(ref_files[name], "resume")
    assert tr.epoch == CC.GAN_EPOCHS_A and tr.total_it == CC.GAN_EPOCHS_A * CC.GAN_ITERS
    assert all(torch.is_tensor(st["step"]) for st in tr.optimizer_g.state.values())
    assert tr.optimizer_g.param_groups[0]["fused"] is fused             # our implementation flag survives the load
    torch.manual_seed(CC.GAN_NOISE_B)
    lrs = []
    while tr.epoch < tr.args.epochs:
        tr.train_epoch(CC.gan_inputs())
        lrs.append((tr.epoch, tr.optimizer_g.param_groups[0]["lr"], tr.optimizer_d.param_groups[0]["lr"]))
    np.testing.assert_allclose(np.array(lrs), golden["gan.lrs"], rtol=1e-15, atol=0)
    assert tr.total_it == int(golden["gan.total_it"])
    for k in ("g_curve", "d_fake_curve", "d_real_curve", "flat_curve"):
        close(getattr(tr, k), golden[f"gan.{k}"], TOL, k)
    t = tr.trainer
    check_states(golden, "gan", (("g", t.generator), ("avg", t.generator_running_avg), ("d", t.discriminator)),
                 (("opt_g", tr.optimizer_g), ("opt_d", tr.optimizer_d)), TOL)


def test_recon_resume_from_reference_checkpoint_continues_the_reference_run(golden, ref_files, monkeypatch):
    """Resume from the reference's checkpoint_2.pth (no 'flat_warmup': the factor restarts at 10, as in the reference) and
    train to epoch 5: every iteration's loss, the per-epoch rates (the network's halves at epoch 4, the DatasetParams' stays),
    the warm-up factor, the network, the DatasetParams and both Adams."""
    _, RT = torch_pieces(monkeypatch)
    tr = recon_trainer(RT, recon_args_b(), CC.RECON_SEED_B)
    tr.flat_warmup.fill_(3.0)
    tr.load_checkpoint(ref_files["recon_ckpt"], "resume")
    assert float(tr.flat_warmup) == 10.0 and tr.epoch == CC.RECON_EPOCHS_A
    losses, lrs = [], []
    while tr.epoch < tr.args.epochs:
        losses += [float(o[0]) for o in tr.train_epoch(CC.recon_batches())]
        lrs.append((tr.epoch, tr.optimizer.param_groups[0]["lr"], tr.optimizer_dataset.param_groups[0]["lr"]))
    np.testing.assert_allclose(np.array(lrs), golden["recon.lrs"], rtol=1e-15, atol=0)
    close(losses, golden["recon.g_curve"], TOL, "losses")
    assert tr.total_it == int(golden["recon.total_it"])
    assert abs(float(tr.flat_warmup) - float(golden["recon.flat_warmup"])) < 1e-5
    check_states(golden, "recon", (("net", tr.generator), ("dp", tr.dataset_params)),
                 (("opt", tr.optimizer), ("opt_dp", tr.optimizer_dataset)), TOL)


def test_recon_resume_restores_flat_warmup_and_evaluate_mode_loads_weights_only(tmp_path, monkeypatch):
    _, RT = torch_pieces(monkeypatch)
    a = recon_args_b()
    tr = recon_trainer(RT, a, CC.RECON_SEED_A)
    tr.train_epoch(CC.recon_batches())
    tr.save_checkpoint(str(tmp_path / "c.pth"))
    fresh = recon_trainer(RT, a, CC.RECON_SEED_B)
    fresh.load_checkpoint(str(tmp_path / "c.pth"), "resume")
    assert torch.equal(fresh.flat_warmup, tr.flat_warmup) and float(fresh.flat_warmup) < 10.0
    ev = recon_trainer(RT, a, CC.RECON_SEED_B)
    ev.load_checkpoint(str(tmp_path / "c.pth"), "evaluate")
    for k, v in tr.generator.state_dict().items():
        assert torch.equal(ev.generator.state_dict()[k], v)
    assert torch.equal(ev.dataset_params.ds_translation, tr.dataset_params.ds_translation)
    assert not ev.optimizer.state and float(ev.flat_warmup) == 10.0 and ev.epoch == 1
    without = recon_trainer(RT, a, CC.RECON_SEED_B, dataset_params=False)
    with pytest.raises(AssertionError):
        without.load_checkpoint(str(tmp_path / "c.pth"), "evaluate")
    with pytest.raises(ValueError):
        ev.load_checkpoint(str(tmp_path / "c.pth"), "continue")


def test_loads_copy_into_the_existing_tensors(golden, ref_files, monkeypatch):
    """Parameters and buffers are restored with load_state_dict's in-place copy: the tensors (and so the pointers a weight
    bank packed) stay the same objects."""
    GT, _ = torch_pieces(monkeypatch)
    tr = gan_trainer(GT, gan_args_b(), CC.GAN_SEED_B)
    mods = (tr.trainer.generator, tr.trainer.generator_running_avg, tr.trainer.discriminator)
    before = [{k: v.data_ptr() for k, v in m.state_dict().items()} for m in mods]
    tr.load_checkpoint(ref_files["gan_ckpt"], "resume")
    ref = CC.decode(golden, "gan_ckpt")
    for m, b, key in zip(mods, before, ("generator", "generator_running_avg", "discriminator")):
        assert {k: v.data_ptr() for k, v in m.state_dict().items()} == b
        for k, v in m.state_dict().items():
            assert torch.equal(v, ref[key][k])


# ------------------------------------------------------------------------------------------------ evaluate mode
def test_gan_evaluate_mode_loads_the_generators_only(golden, ref_files, monkeypatch):
    GT, _ = torch_pieces(monkeypatch)
    tr = gan_trainer(GT, gan_args_b(), CC.GAN_SEED_B)
    d_before = {k: v.clone() for k, v in tr.trainer.discriminator.state_dict().items()}
    tr.load_checkpoint(ref_files["gan_ckpt"], "evaluate")
    ref = CC.decode(golden, "gan_ckpt")
    for k, v in tr.trainer.generator_running_avg.state_dict().items():
        assert torch.equal(v, ref["generator_running_avg"][k])
    for k, v in tr.trainer.generator.state_dict().items():
        assert torch.equal(v, ref["generator"][k])
    for k, v in tr.trainer.discriminator.state_dict().items():
        assert torch.equal(v, d_before[k])
    assert not tr.optimizer_g.state and not tr.optimizer_d.state


def test_evaluate_mode_loads_a_running_average_only_file_with_the_shipped_layout(tmp_path):
    """The shipped gan_weights/*/checkpoint_latest.pth holds only 'generator_running_avg' (512², three discriminators; its
    names and shapes are pinned in reference_pins.npz): it loads, and the live generator is left as it was."""
    from gan_training import GANTrainer
    pins = np.load(os.path.join(GOLDEN, "reference_pins.npz"))
    import bench
    args = bench.gan_args(512, 3)
    tr = GANTrainer(args, device="cpu")
    g = torch.Generator().manual_seed(1)
    sd = {}
    for name, shape, v in zip(pins["ckpt_names"], pins["ckpt_shapes"], tr.trainer.generator_running_avg.state_dict().values()):
        shape = tuple(int(s) for s in str(shape).split(",") if s)
        assert tuple(v.shape) == shape
        sd[str(name)] = (torch.randn(shape, generator=g) if v.is_floating_point() else torch.full(shape, 5, dtype=v.dtype))
    torch.save({"generator_running_avg": sd}, str(tmp_path / "checkpoint_latest.pth"))
    g_before = {k: v.clone() for k, v in tr.trainer.generator.state_dict().items()}
    tr.load_checkpoint(str(tmp_path / "checkpoint_latest.pth"), "evaluate")
    for k, v in tr.trainer.generator_running_avg.state_dict().items():
        assert torch.equal(v, sd[k])
    for k, v in tr.trainer.generator.state_dict().items():
        assert torch.equal(v, g_before[k])
    assert tr.epoch == 0 and tr.total_it == 0


# ------------------------------------------------------------------------------------------------ best-epoch search
class StandInEvaluator:
    def __init__(self, avg):
        self.avg, self.calls = avg, []

    def evaluate(self, batches, fast=False, seed=None, distributed=False):
        self.calls.append((int(round(float(self.avg.fc.bias[0].detach()))), fast, seed, distributed))
        return {"fid": CC.search_fid(self.avg)}


def test_best_epoch_search_matches_the_reference_search(golden, tmp_path, monkeypatch):
    """Newest epoch first, numerically (100 before 40), checkpoint_latest.pth skipped; ties do not replace the best; the
    best checkpoint is loaded again for the full evaluation."""
    from fid_evaluation import select_best_checkpoint
    GT, _ = torch_pieces(monkeypatch)
    CC.write_search_checkpoints(str(tmp_path))
    tr = gan_trainer(GT, gan_args_b(), CC.GAN_SEED_B)
    ev = StandInEvaluator(tr.trainer.generator_running_avg)
    out = select_best_checkpoint(tr, ev, str(tmp_path), [], seed=1234)
    visited = [c[0] for c in ev.calls]
    assert visited[:-1] == golden["search.visited"].tolist() and all(c[1] for c in ev.calls[:-1])
    assert list(out["fast_fid"]) == visited[:-1] and list(out["fast_fid"].values()) == [CC.SEARCH_FID[e] for e in visited[:-1]]
    assert os.path.basename(out["best_path"]) == str(golden["search.best"])
    assert ev.calls[-1] == (int(golden["search.final_loaded"]), False, 1234, False)
    assert out["scores"]["fid"] == CC.SEARCH_FID[int(golden["search.final_loaded"])]
    assert float(tr.trainer.generator.fc.bias[0].detach()) == -int(golden["search.final_loaded"])
    open(str(tmp_path / "checkpoint_7b.pth"), "wb").close()
    with pytest.raises(ValueError, match="Invalid path"):
        select_best_checkpoint(tr, ev, str(tmp_path), [])


# ------------------------------------------------------------------------------------------------ torch.distributed
def _snapshot(tr):
    """numpy copies (a torch tensor put on a multiprocessing queue is shared with, not copied from, the exiting worker)."""
    t = tr.trainer
    out = {f"{n}.{k}": v for n, m in (("g", t.generator), ("avg", t.generator_running_avg), ("d", t.discriminator))
           for k, v in m.state_dict().items()}
    out.update({f"opt_g.{k}": v for k, v in CC.adam_state(tr.optimizer_g).items()})
    out.update({f"opt_d.{k}": v for k, v in CC.adam_state(tr.optimizer_d).items()})
    out = {k: v.detach().cpu().numpy().copy() for k, v in out.items()}
    return out, (tr.epoch, tr.total_it, tr.g_curve, tr.d_fake_curve, tr.d_real_curve, tr.flat_curve)


def _worker(rank, world, port, path, q):
    for p in (PKG, ROOT, GOLDEN, os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    mp_ = pytest.MonkeyPatch()
    try:
        GT, _ = torch_pieces(mp_)
        tr = gan_trainer(GT, gan_args_b(), CC.GAN_SEED_A + rank)          # the ranks start from different states
        torch.manual_seed(rank)
        tr.train_epoch(CC.gan_inputs()[:2 + rank])
        saved = _snapshot(tr)
        tr.save_checkpoint(path)                                          # rank 0 writes; both wait at the barrier
        fresh = gan_trainer(GT, gan_args_b(), 40 + rank)
        fresh.load_checkpoint(path, "resume")
        q.put((rank, saved, _snapshot(fresh)))
    finally:
        mp_.undo()
    dist.barrier()
    dist.destroy_process_group()


def test_rank0_saves_and_every_rank_loads_the_same_state(tmp_path):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35000 + os.getpid() % 2000
    path = str(tmp_path / "checkpoint_latest.pth")
    procs = [ctx.Process(target=_worker, args=(r, 2, port, path, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict((r, (s, l)) for r, s, l in [q.get(timeout=180) for _ in procs])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (saved0, meta0), _ = res[0]
    for rank in (0, 1):
        loaded, meta = res[rank][1]
        assert meta == meta0 and set(loaded) == set(saved0)
        for k, v in loaded.items():
            assert v.dtype == saved0[k].dtype and np.array_equal(v, saved0[k]), (rank, k)
    assert not all(np.array_equal(res[1][0][0][k], saved0[k]) for k in saved0)   # rank 1's own state was different
