"""Generate tests/golden/drivers_reference.npz from the reference's two scripts (authoring container only):
    python tests/golden/make_golden_drivers.py
main.py and run_reconstruction.py parse their command line at import time, so nothing is imported from them.  Taken from
their syntax trees and executed unmodified:
  * the parsers: `parser = argparse.ArgumentParser()` and every module-level `parser.add_argument(...)`.  Recorded: every
    flag's option strings, dest, default, type, action class and `required`, and for every argv sample (the README's
    commands and the quirks) the parsed namespace or the fact that argparse exits with an error;
  * main.py's derived settings (:88-121, from `cache_dir = ...` to the safety checks), run with the working directory
    set to dataset_common.write_tree's synthetic caches against the reference's dataset classes, for cub / p3d x
    256 / 512 x --conditional_color, plus three discriminators at 256: mesh path, number of discriminators, truncation
    sigma, or the assertion that fails;
  * the training loops, through make_golden_checkpoint.py's namespaces (stand-in networks and batches) with
    args.tensorboard on: every log() line and every add_scalar call of the epochs that run;
  * the format strings of every log('...'.format(...)) call (the FID, '[TEST]' and epoch-time lines);
  * the best-epoch search (:787-830) on checkpoint_common's search checkpoints: the lines it prints.
Nothing of the reference is copied into the repository, only its outputs and the text of its log lines."""
import argparse
import ast
import json
import os
import sys
import tempfile

import numpy as np
import torch

REF = "/root/reference/code"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, REF)
import checkpoint_common as CC                                 # noqa: E402
import dataset_common as DC                                    # noqa: E402
import make_golden_checkpoint as MC                            # noqa: E402

README_MAIN = [
    "--dataset cub --batch_size 16 --weights pretrained_weights_cub --save_results",
    "--dataset p3d --batch_size 16 --weights pretrained_weights_p3d --save_results",
    "--dataset cub --batch_size 16 --weights pretrained_weights_cub",
    "--dataset p3d --batch_size 16 --weights pretrained_weights_p3d",
    "--name cub_512x512_class --conditional_class --dataset cub --gpu_ids 0,1,2,3 --batch_size 32 --epochs 1000 --tensorboard",
    "--name cub_512x512_class --conditional_class --dataset cub --gpu_ids 0,1,2,3 --batch_size 64 --evaluate --which_epoch best",
]
EXTRA_MAIN = [
    "--weights w --dataset cub --symmetric_g False",
    "--weights w --dataset cub --symmetric_g ''",
    "--weights w --dataset cub --continue_train --which_epoch best",
    "--weights w --dataset p3d --conditional_color --texture_resolution 256 --truncation_sigma 0.5 --norm_g instance",
    "--weights w",
    "--dataset cub",
    "--weights w --dataset cub --epochs ten",
]
README_RECON = [
    "--name pretrained_reconstruction_cub --dataset cub --batch_size 10 --generate_pseudogt",
    "--name pretrained_reconstruction_p3d --dataset p3d --optimize_z0 --batch_size 10 --generate_pseudogt",
    "--name pretrained_reconstruction_cub --dataset cub --batch_size 50 --tensorboard",
    "--name pretrained_reconstruction_p3d --dataset p3d --optimize_z0 --batch_size 50 --tensorboard",
]
EXTRA_RECON = [
    "--name r --dataset cub --symmetric False",
    "--name r --dataset cub --symmetric ''",
    "--name r --dataset cub --continue_train --which_epoch best",
    "--name r --dataset cub --generate_pseudogt --optimize_z0 --pseudogt_resolution 256",
    "--name r --dataset cub --optimize_deltas '' --loss l1 --lr 0.001",
    "--name r",
    "--name r --dataset cub --gpu_ids 0",
]
DERIVED = [f"--weights w --dataset {ds} --evaluate --texture_resolution {r}" + (" --conditional_color" if cc else "")
           for ds in ("cub", "p3d") for r in (256, 512) for cc in (False, True)]
DERIVED.append("--weights w --dataset cub --evaluate --texture_resolution 256 --num_discriminators 3")


def split(line):
    import shlex
    return shlex.split(line)


def reference_parser(src):
    tree = ast.parse(src)
    nodes = [n for n in tree.body
             if (isinstance(n, ast.Assign) and ast.get_source_segment(src, n) == "parser = argparse.ArgumentParser()")
             or (isinstance(n, ast.Expr) and ast.get_source_segment(src, n).startswith("parser.add_argument("))]
    ns = {"argparse": argparse}
    exec(compile(ast.Module(body=nodes, type_ignores=[]), "parser", "exec"), ns)
    return ns["parser"]


def describe(parser):
    out = []
    for a in parser._actions:
        if isinstance(a, argparse._HelpAction):
            continue
        out.append(dict(option_strings=a.option_strings, dest=a.dest, default=repr(a.default),
                        type=getattr(a.type, "__name__", None), action=type(a).__name__, required=a.required))
    return out


def parse(parser, argv):
    try:
        with open(os.devnull, "w") as null:
            old, sys.stderr = sys.stderr, null
            try:
                return {k: repr(v) for k, v in sorted(vars(parser.parse_args(argv)).items())}
            finally:
                sys.stderr = old
    except SystemExit:
        return "error"


def format_strings(src):
    """The '...' of every log('...'.format(...)) call."""
    out = []
    for n in ast.walk(ast.parse(src)):
        if (isinstance(n, ast.Call) and isinstance(n.func, ast.Name) and n.func.id == "log" and n.args
                and isinstance(n.args[0], ast.Call) and isinstance(n.args[0].func, ast.Attribute)
                and isinstance(n.args[0].func.value, ast.Constant)):
            out.append(n.args[0].func.value.value)
    return out


def derived(src, parser):
    tree = ast.parse(src)
    body = tree.body
    a = next(i for i, n in enumerate(body) if ast.get_source_segment(src, n) == "cache_dir = os.path.join('cache', args.dataset)")
    b = next(i for i, n in enumerate(body) if isinstance(n, ast.If) and ast.get_source_segment(src, n.test) == "args.norm_g == 'syncbatch'")
    block = compile(ast.Module(body=body[a:b], type_ignores=[]), "main.py", "exec")
    out = []
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as root:
        DC.write_tree(root, DC.make_inputs())
        os.chdir(root)
        try:
            for line in DERIVED:
                args = parser.parse_args(split(line))
                try:
                    exec(block, {"os": os, "args": args})
                    out.append(dict(mesh_path=args.mesh_path, num_discriminators=args.num_discriminators,
                                    truncation_sigma=args.truncation_sigma, error=None))
                except AssertionError as e:
                    out.append(dict(error=f"AssertionError: {e}"))
        finally:
            os.chdir(cwd)
    return out


class Writer:
    def __init__(self):
        self.scalars = []

    def add_scalar(self, tag, value, step):
        self.scalars.append((tag, float(value), int(step)))


def gan_loop(src, tree):
    loop = MC._compile(src, [MC._while(tree, "optimizer_g")], "main.py")
    a = CC.gan_args()
    a.epochs, a.lr_decay_after, a.save_freq, a.checkpoint_freq, a.evaluate_freq = 3, 1000, 1, 100, 100
    a.continue_train, a.which_epoch, a.tensorboard = False, "latest", True
    lines, w = [], Writer()
    with tempfile.TemporaryDirectory() as d:
        ns = MC.gan_namespace(src, tree, a, CC.GAN_SEED_A, d, [])
        ns.update(log=lines.append, writer=w)
        torch.manual_seed(CC.GAN_NOISE_A)
        exec(loop, ns)
    return dict(lines=lines, scalars=w.scalars, epochs=a.epochs, n_iters=len(ns["train_loader"]),
                d_steps_per_g=a.d_steps_per_g, loss=a.loss)


def recon_loop(tree):
    src = open(os.path.join(REF, "run_reconstruction.py")).read()
    tree = ast.parse(src)
    loop = MC._compile(src, [MC._while(tree, "recon_loss")], "run_reconstruction.py")
    a = CC.recon_args()
    a.epochs, a.lr_decay_every, a.save_freq, a.checkpoint_freq, a.evaluate_freq = 3, 1000, 1, 100, 100
    a.tensorboard, a.image_freq = True, 100
    lines, w = [], Writer()
    with tempfile.TemporaryDirectory() as d:
        ns = MC.recon_namespace(tree, a, CC.RECON_SEED_A, d, [])
        ns.update(log=lines.append, writer=w)
        exec(loop, ns)
    return dict(lines=lines, scalars=w.scalars, total=list(ns["g_curve"]), n_iters=len(ns["train_loader"]), loss=a.loss)


def search(src, tree):
    """main.py:787-830 (`if args.which_epoch == 'best':`) on checkpoint_common's search checkpoints, with its print()
    lines captured; the stand-in evaluate_fid logs the fast evaluation's FID line as the reference's does.  The
    checkpoint directory is 'w', relative to the working directory, so that the printed paths do not depend on it."""
    import glob
    import wrapper_common as WC
    block = MC._compile(src, [MC._if(tree, "args.which_epoch == 'best'", src, "best_fid")], "main.py")
    gi, _ = WC.build()
    G, avg = gi(), gi()
    lines = []

    def evaluate_fid(writer, it, idx=None, fast=False):
        fid = CC.search_fid(avg)
        lines.append('FID (training set): {:.02f}'.format(fid))
        return fid
    args = CC.gan_args()
    args.which_epoch = "best"
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, "w"))
        CC.write_search_checkpoints(os.path.join(d, "w"))
        os.chdir(d)
        try:
            ns = {"torch": torch, "os": os, "glob": glob, "args": args, "checkpoint_dir": "w", "generator": G,
                  "generator_running_avg": avg, "evaluate_fid": evaluate_fid, "writer": None, "total_it": 0,
                  "print": lambda *x: lines.append(" ".join(str(v) for v in x))}
            exec(block, ns)
        finally:
            os.chdir(cwd)
    return dict(lines=lines, fast_fid=[[e, CC.SEARCH_FID[e]] for e in sorted(CC.SEARCH_FID, reverse=True)],
                best_path=ns["best_checkpoint"])


def main():
    main_src = open(os.path.join(REF, "main.py")).read()
    recon_src = open(os.path.join(REF, "run_reconstruction.py")).read()
    pm, pr = reference_parser(main_src), reference_parser(recon_src)
    out = dict(
        main_flags=describe(pm), recon_flags=describe(pr),
        main_samples=[[s, parse(pm, split(s))] for s in README_MAIN + EXTRA_MAIN],
        recon_samples=[[s, parse(pr, split(s))] for s in README_RECON + EXTRA_RECON],
        derived=[[s, d] for s, d in zip(DERIVED, derived(main_src, pm))],
        main_formats=format_strings(main_src), recon_formats=format_strings(recon_src),
        gan_loop=gan_loop(main_src, ast.parse(main_src)), recon_loop=recon_loop(None),
        search=search(main_src, ast.parse(main_src)),
    )
    p = os.path.join(HERE, "drivers_reference.npz")
    np.savez_compressed(p, json=np.array(json.dumps(out)))
    print("wrote", p, os.path.getsize(p), "bytes")
    print(json.dumps({k: out[k] for k in ("derived", "main_formats", "recon_formats")}, indent=1)[:3000])
    print(out["gan_loop"]["lines"][:3], out["recon_loop"]["lines"][:3])


if __name__ == "__main__":
    main()
