"""Generate tests/golden/recon_eval_reference.npz by EXECUTING the reference's validation pass, turntable render and L1
training iteration, and its reconstruction network in eval mode (authoring container only):
    python tests/golden/make_golden_recon_eval.py
It reads no other golden and runs on its own, beside regenerate_all.sh (which does not list it).  As in make_golden_recon_step.py, functions are taken from run_reconstruction.py's syntax tree and compiled unmodified:
`mean_iou` (:225-231), `transform_vertices` (:237-252), `evaluate_all` (:255-319), `render_multiview` (:188-221) and the
training loop (:409-465).  The namespace provides the module globals they read, with recon_step_common.py's stand-ins for
the network, template and renderer; `.cuda()` is the identity.
  * evaluate_all, writer=None, for criterion nn.MSELoss() / nn.L1Loss() (:347-352) x {deltas, z0, deltas + z0}, on a
    stand-in network with seeded batch-norm running statistics and seeded DatasetParams (recon_eval_common.py).  Stored:
    the '[TEST] ...' log line and the fp64 totals, read from the function's locals when it returns (a profile hook; the
    function itself is unchanged).
  * render_multiview on one stand-in prediction: the [2R, 4R, 3] tile and its inputs.
  * the training loop with criterion = nn.L1Loss(), four iterations: the fields of recon_step_reference.npz.
  * models/reconstruction.py imported unmodified, built by recon_common.build, with recon_eval_common's running
    statistics: one .eval() forward on recon_common.inputs() -> texture probe, texture sum, displacement map.
Nothing of the reference is copied into the repository — only its outputs."""
import ast
import os
import sys
import time

import numpy as np
import torch
import torch.nn as nn
import torch.optim as optim

REF = "/root/reference/code"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, REF)
import recon_common as RC                                      # noqa: E402
import recon_eval_common as RE                                 # noqa: E402
import recon_step_common as RS                                 # noqa: E402
from make_golden_recon_step import find_loop                   # noqa: E402
from models import reconstruction as ref_recon                 # noqa: E402  (reference)
from models.reconstruction import DatasetParams               # noqa: E402  (reference)
from rendering.utils import qmul, qrot                        # noqa: E402  (reference)
from utils.losses import loss_flat                            # noqa: E402  (reference)

torch.Tensor.cuda = lambda self, *a, **k: self

CRITERIA = {"mse": nn.MSELoss, "l1": nn.L1Loss}


def script_functions(*names):
    tree = ast.parse(open(os.path.join(REF, "run_reconstruction.py")).read())
    funcs = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert len(funcs) == len(names)
    return tree, funcs


def namespace(args, generator, dataset_params, criterion, logs):
    return {"torch": torch, "np": np, "qrot": qrot, "qmul": qmul, "args": args, "generator": generator,
            "dataset_params": dataset_params, "criterion": criterion, "loss_flat": loss_flat,
            "mesh_template": RS.Template(), "renderer": None, "log": logs.append}


def eval_args(deltas, z0, loss):
    args = RS.make_args(deltas, z0)
    args.loss, args.batch_size, args.image_resolution = loss, 4, RS.H
    return args


def run_evaluate(deltas, z0, loss):
    _, funcs = script_functions("mean_iou", "transform_vertices", "evaluate_all")
    args = eval_args(deltas, z0, loss)
    generator = RE.set_running_stats(RS.build_net())
    dp = RE.perturb_dataset_params(DatasetParams(args, 10))
    logs = []
    ns = namespace(args, generator, dp, CRITERIA[loss](), logs)
    exec(compile(ast.Module(body=funcs, type_ignores=[]), "run_reconstruction.py", "exec"), ns)
    totals = {}

    def hook(frame, event, arg):
        if event == "return" and frame.f_code.co_name == "evaluate_all":
            totals.update({k: frame.f_locals[k] for k in ("total_recon_loss", "total_flat_loss", "total_miou", "N")})
    sys.setprofile(hook)
    try:
        ns["evaluate_all"](RE.eval_batches())
    finally:
        sys.setprofile(None)
    assert len(logs) == 1 and not generator.training
    return {"log": np.array(logs[0]), "totals": np.array([totals["total_recon_loss"], totals["total_flat_loss"],
                                                          totals["total_miou"], totals["N"]], dtype=np.float64)}


def run_multiview():
    _, funcs = script_functions("render_multiview")
    args = eval_args(True, False, "mse")
    X = RE.eval_batches()[0][0]
    tpl = RS.Template()
    with torch.no_grad():
        pred_tex, mesh_map = RE.set_running_stats(RS.build_net()).eval()(X)
        raw_vtx = tpl.get_vertex_positions(mesh_map)
    ns = namespace(args, None, None, None, [])
    exec(compile(ast.Module(body=funcs, type_ignores=[]), "run_reconstruction.py", "exec"), ns)
    tile = ns["render_multiview"](raw_vtx, pred_tex, RE.MULTIVIEW_IDX)
    return {"raw_vtx": raw_vtx.numpy(), "pred_tex": pred_tex.numpy(), "tile": tile}


def run_l1_loop(deltas, z0):
    tree, funcs = script_functions("mean_iou", "transform_vertices")
    args = RS.make_args(deltas, z0)
    args.loss = "l1"
    generator = RS.build_net().train()
    dataset_params = DatasetParams(args, 10)
    logs = []
    ns = namespace(args, generator, dataset_params, nn.L1Loss(), logs)
    ns.update({"optimizer": optim.Adam(generator.parameters(), lr=args.lr),
               "optimizer_dataset": optim.Adam(dataset_params.parameters(), lr=args.lr_dataset),
               "train_loader": RS.batches(), "flat_warmup": 10, "g_curve": [], "total_it": 0, "epoch": 0, "time": time})
    exec(compile(ast.Module(body=funcs + [find_loop(tree)], type_ignores=[]), "run_reconstruction.py", "exec"), ns)
    assert ns["total_it"] == 4 and len(logs) == 1
    out = {"g_curve": np.array(ns["g_curve"]), "flat_warmup": np.float64(ns["flat_warmup"]), "log0": np.array(logs[0])}
    for k, v in generator.state_dict().items():
        out["net." + k] = v.numpy().copy()
    for k, v in dataset_params.state_dict().items():
        out["dp." + k] = v.numpy().copy()
    return out


def run_eval_network():
    torch.set_num_threads(8)
    net = RE.set_running_stats(RC.build(ref_recon)).eval()
    x, _, _ = RC.inputs()
    with torch.no_grad():
        tex, mesh_map = net(x)
    return {"tex_probe": tex[:, :, ::8, ::8].numpy(), "tex_sum": np.float64(tex.double().sum()), "mesh_map": mesh_map.numpy()}


def main():
    out = {}
    for loss in RE.CRITERIA:
        for tag, deltas, z0 in RE.POSES:
            for k, v in run_evaluate(deltas, z0, loss).items():
                out[f"eval.{loss}.{tag}.{k}"] = v
    for k, v in run_multiview().items():
        out["multiview." + k] = v
    for tag, deltas, z0 in RE.POSES:
        for k, v in run_l1_loop(deltas, z0).items():
            out[f"l1step.{tag}.{k}"] = v
    for k, v in run_eval_network().items():
        out["evalnet." + k] = v
    p = os.path.join(HERE, "recon_eval_reference.npz")
    np.savez_compressed(p, **out)
    print("wrote", p, os.path.getsize(p), "bytes")
    for k, v in out.items():
        if k.endswith(".log") or k.endswith(".totals") or k.endswith("g_curve") or k.endswith("log0") or k.endswith("tex_sum"):
            print(" ", k, v.tolist())


if __name__ == "__main__":
    main()
