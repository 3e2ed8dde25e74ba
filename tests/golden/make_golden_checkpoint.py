"""Generate the checkpoint goldens by EXECUTING the reference's epoch layer (authoring container only):
    python tests/golden/make_golden_checkpoint.py
main.py and run_reconstruction.py cannot be imported.  Taken from their syntax trees and compiled unmodified:
  * main.py: `divide_pred`, `update_generator_running_avg`, `ModelWrapper` (execution patch D15, as make_golden_gan_loop.py),
    the loading block `if args.continue_train or args.evaluate:` (:599-633), the training `while epoch < args.epochs:` loop
    (:670-782: iterations, epoch counter, linear learning-rate decay, the save_checkpoint closure) and the
    `if args.which_epoch == 'best':` search (:787-830);
  * run_reconstruction.py: `mean_iou`, `transform_vertices`, the loading block `if args.evaluate or args.generate_pseudogt:`
    (:359-382) and the training `while` loop (:407-490: iterations, learning-rate halving, save_checkpoint).
The stand-in networks, template and renderer are those of wrapper_common.py / recon_step_common.py; the settings and
batches are checkpoint_common.py's.  `evaluate_fid` / `evaluate_all` are stand-ins that record the learning rates the epoch
ends with (the search's evaluate_fid scores with checkpoint_common.search_fid).

Writes tests/golden/checkpoint_reference.npz:
  gan_ckpt.*          the GAN checkpoint_2.pth run A wrote (checkpoint_common.encode: manifest + tensors);
  gan_ckpt_numstep.*  the same with every Adam `step` a Python int, as torch < 1.12 wrote it;
  recon_ckpt.*        the reconstruction checkpoint_2.pth run A wrote;
  gan.* / recon.*     run B of each (resumed from those files): curves, learning rates per epoch, iteration counter,
                      final parameters / buffers / Adam state;
  search.*            the search's visit order and choice.
Nothing of the reference is copied into the repository, only its outputs."""
import ast
import glob
import math
import os
import sys
import tempfile
import time

import numpy as np
import torch
import torch.nn as nn
import torch.optim as optim

REF = "/root/reference/code"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, REF)
import checkpoint_common as CC                                 # noqa: E402
import recon_step_common as RS                                 # noqa: E402
import wrapper_common as WC                                    # noqa: E402
from models.reconstruction import DatasetParams               # noqa: E402  (reference)
from rendering.utils import qrot                              # noqa: E402  (reference)
from utils.losses import GANLoss, loss_flat                    # noqa: E402  (reference)

torch.Tensor.cuda = lambda self, *a, **k: self                 # D15


def _compile(src, nodes, name):
    return compile(ast.Module(body=nodes, type_ignores=[]), name, "exec")


def _while(tree, marker):
    return next(n for n in ast.walk(tree) if isinstance(n, ast.While) and marker in ast.dump(n))


def _if(tree, test_src, src, marker=""):
    return next(n for n in ast.walk(tree) if isinstance(n, ast.If) and ast.get_source_segment(src, n.test) == test_src
                and marker in ast.dump(n))


def store(out, prefix, tensors):
    for k, v in tensors.items():
        out[f"{prefix}.{k}"] = v.detach().cpu().numpy().copy()


# ------------------------------------------------------------------------------------------------ GAN
def gan_namespace(src, tree, args, seed, ckdir, lrs):
    defs = [n for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and
            n.name in ("divide_pred", "update_generator_running_avg", "ModelWrapper")]
    seg = "\n\n".join(ast.get_source_segment(src, n) for n in defs)
    patched = seg.replace("GANLoss(args.loss, tensor=torch.cuda.FloatTensor).cuda()", "GANLoss(args.loss, tensor=torch.FloatTensor)")
    assert len(defs) == 3 and patched != seg
    ns = {"torch": torch, "nn": nn, "math": math, "os": os, "GANLoss": GANLoss, "args": args}
    exec(compile(patched, "main.py", "exec"), ns)
    gi, D = WC.build(seed)
    trainer = ns["ModelWrapper"](gi, D).train()

    def evaluate_fid(writer, it, idx=None, fast=False):
        lrs.append((ns["epoch"], ns["optimizer_g"].param_groups[0]["lr"], ns["optimizer_d"].param_groups[0]["lr"]))
    ns.update(trainer=trainer, generator=trainer.generator, generator_running_avg=trainer.generator_running_avg,
              discriminator=trainer.discriminator,
              optimizer_g=optim.Adam(trainer.generator.parameters(), lr=args.lr_g, betas=(0.0, 0.9)),
              optimizer_d=optim.Adam(trainer.discriminator.parameters(), lr=args.lr_d, betas=(0.0, 0.9)),
              mesh_template=RS.Template(map_size=8), loss_flat=loss_flat, use_mesh=True, train_loader=CC.gan_loader(),
              d_fake_curve=[0], d_real_curve=[0], g_curve=[0], flat_curve=[0], total_it=0, epoch=0, time=time,
              log=lambda s: None, writer=None, checkpoint_dir=ckdir, evaluate_fid=evaluate_fid)
    return ns


def gan(out, ckdir):
    src = open(os.path.join(REF, "main.py")).read()
    tree = ast.parse(src)
    loop = _compile(src, [_while(tree, "optimizer_g")], "main.py")
    load = _compile(src, [_if(tree, "args.continue_train or args.evaluate", src)], "main.py")
    # run A: epochs 0-1 from scratch
    a = CC.gan_args()
    a.epochs, a.lr_decay_after, a.save_freq, a.checkpoint_freq, a.evaluate_freq = CC.GAN_EPOCHS_A, 1000, 1, 1, 1
    a.continue_train, a.which_epoch = False, "latest"
    ns = gan_namespace(src, tree, a, CC.GAN_SEED_A, ckdir, [])
    torch.manual_seed(CC.GAN_NOISE_A)
    exec(loop, ns)
    chk = torch.load(os.path.join(ckdir, f"checkpoint_{CC.GAN_EPOCHS_A}.pth"))
    CC.encode(chk, "gan_ckpt", out)
    for k in ("optimizer_g", "optimizer_d"):
        for st in chk[k]["state"].values():
            st["step"] = int(st["step"])
    CC.encode(chk, "gan_ckpt_numstep", out)
    # run B: --continue_train --which_epoch 2, to epoch 6 with the decay from epoch 3
    b = CC.gan_args()
    b.epochs, b.lr_decay_after, b.save_freq, b.checkpoint_freq, b.evaluate_freq = CC.GAN_EPOCHS_B, CC.GAN_DECAY_AFTER_B, 1, 100, 1
    b.continue_train, b.which_epoch, b.evaluate = True, str(CC.GAN_EPOCHS_A), False
    lrs = []
    ns = gan_namespace(src, tree, b, CC.GAN_SEED_B, ckdir, lrs)
    ns["print"] = lambda *x: None
    exec(load, ns)
    assert ns["epoch"] == CC.GAN_EPOCHS_A and ns["total_it"] == CC.GAN_EPOCHS_A * CC.GAN_ITERS
    torch.manual_seed(CC.GAN_NOISE_B)
    exec(loop, ns)
    for k in ("g_curve", "d_fake_curve", "d_real_curve", "flat_curve"):
        out[f"gan.{k}"] = np.array(ns[k], dtype=np.float64)
    out["gan.lrs"] = np.array(lrs, dtype=np.float64)
    out["gan.total_it"] = np.int64(ns["total_it"])
    for name, mod in (("g", ns["generator"]), ("avg", ns["generator_running_avg"]), ("d", ns["discriminator"])):
        store(out, f"gan.{name}", mod.state_dict())
    store(out, "gan.opt_g", CC.adam_state(ns["optimizer_g"]))
    store(out, "gan.opt_d", CC.adam_state(ns["optimizer_d"]))
    return src, tree


# ------------------------------------------------------------------------------------------------ reconstruction
def recon_namespace(tree, args, seed, ckdir, lrs):
    funcs = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in ("mean_iou", "transform_vertices")]
    assert len(funcs) == 2
    generator = RS.build_net(seed).train()
    torch.manual_seed(seed)
    dataset_params = DatasetParams(args, 10)
    with torch.no_grad():                   # DatasetParams start at zero / one: make run B's differ from run A's
        for p in dataset_params.parameters():
            p.add_(0.01 * torch.randn(p.shape))
    ns = {"torch": torch, "os": os, "qrot": qrot, "args": args, "generator": generator, "dataset_params": dataset_params,
          "optimizer": optim.Adam(generator.parameters(), lr=args.lr),
          "optimizer_dataset": optim.Adam(dataset_params.parameters(), lr=args.lr_dataset),
          "criterion": nn.MSELoss(), "loss_flat": loss_flat, "mesh_template": RS.Template(), "renderer": None,
          "train_loader": RS.batches(), "flat_warmup": 10, "g_curve": [], "total_it": 0, "epoch": 0, "time": time,
          "log": lambda s: None, "writer": None, "val_loader": None, "checkpoint_dir": ckdir, "print": lambda *x: None}

    def evaluate_all(loader, writer, it):
        lrs.append((ns["epoch"], ns["optimizer"].param_groups[0]["lr"], ns["optimizer_dataset"].param_groups[0]["lr"]))
    ns["evaluate_all"] = evaluate_all
    exec(_compile(None, funcs, "run_reconstruction.py"), ns)
    return ns


def recon(out, ckdir):
    src = open(os.path.join(REF, "run_reconstruction.py")).read()
    tree = ast.parse(src)
    loop = _compile(src, [_while(tree, "recon_loss")], "run_reconstruction.py")
    load = _compile(src, [_if(tree, "args.evaluate or args.generate_pseudogt", src)], "run_reconstruction.py")
    a = CC.recon_args()
    a.epochs, a.lr_decay_every, a.save_freq, a.checkpoint_freq, a.evaluate_freq = CC.RECON_EPOCHS_A, CC.RECON_DECAY_EVERY, 1, 1, 1
    ns = recon_namespace(tree, a, CC.RECON_SEED_A, ckdir, [])
    exec(loop, ns)
    CC.encode(torch.load(os.path.join(ckdir, f"checkpoint_{CC.RECON_EPOCHS_A}.pth")), "recon_ckpt", out)
    # run B: the reference resumes only under --evaluate (or --generate_pseudogt) together with --continue_train (SURVEY
    # App. A D16); the warm-up factor restarts at 10
    b = CC.recon_args()
    b.epochs, b.lr_decay_every, b.save_freq, b.checkpoint_freq, b.evaluate_freq = CC.RECON_EPOCHS_B, CC.RECON_DECAY_EVERY, 1, 100, 1
    b.evaluate, b.generate_pseudogt, b.continue_train, b.which_epoch = True, False, True, str(CC.RECON_EPOCHS_A)
    lrs = []
    ns = recon_namespace(tree, b, CC.RECON_SEED_B, ckdir, lrs)
    exec(load, ns)
    assert ns["epoch"] == CC.RECON_EPOCHS_A
    exec(loop, ns)
    out["recon.g_curve"] = np.array(ns["g_curve"], dtype=np.float64)
    out["recon.lrs"] = np.array(lrs, dtype=np.float64)
    out["recon.total_it"] = np.int64(ns["total_it"])
    out["recon.flat_warmup"] = np.float64(ns["flat_warmup"])
    store(out, "recon.net", ns["generator"].state_dict())
    store(out, "recon.dp", ns["dataset_params"].state_dict())
    store(out, "recon.opt", CC.adam_state(ns["optimizer"]))
    store(out, "recon.opt_dp", CC.adam_state(ns["optimizer_dataset"]))


# ------------------------------------------------------------------------------------------------ best-epoch search
def search(out, src, tree, ckdir):
    CC.write_search_checkpoints(ckdir)
    block = _compile(src, [_if(tree, "args.which_epoch == 'best'", src, "best_fid")], "main.py")
    gi, _ = WC.build()
    G, avg = gi(), gi()
    visited = []

    def evaluate_fid(writer, it, idx=None, fast=False):
        assert fast
        visited.append(int(round(float(avg.fc.bias[0]))))
        assert float(G.fc.bias[0]) == -visited[-1]
        return CC.search_fid(avg)
    args = CC.gan_args()
    args.which_epoch = "best"
    ns = {"torch": torch, "os": os, "glob": glob, "args": args, "checkpoint_dir": ckdir, "generator": G,
          "generator_running_avg": avg, "evaluate_fid": evaluate_fid, "writer": None, "total_it": 0, "print": lambda *x: None}
    exec(block, ns)
    out["search.visited"] = np.array(visited, dtype=np.int64)
    out["search.best"] = np.array(os.path.basename(ns["best_checkpoint"]))
    out["search.final_loaded"] = np.int64(round(float(avg.fc.bias[0])))


def main():
    out = {}
    with tempfile.TemporaryDirectory() as d1, tempfile.TemporaryDirectory() as d2, tempfile.TemporaryDirectory() as d3:
        src, tree = gan(out, d1)
        recon(out, d2)
        search(out, src, tree, d3)
    p = os.path.join(HERE, "checkpoint_reference.npz")
    np.savez_compressed(p, **out)
    print("wrote", p, os.path.getsize(p), "bytes")
    print({k: out[k].tolist() for k in ("gan.lrs", "recon.lrs", "search.visited", "search.best", "gan.total_it")})


if __name__ == "__main__":
    main()
