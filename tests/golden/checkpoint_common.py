"""Shared by make_golden_checkpoint.py (reference side) and tests/test_checkpoint_hostlogic.py (drop-in side): the settings,
batches and search fixtures of the checkpoint goldens, on the stand-ins of wrapper_common.py / recon_step_common.py.

GAN: 4 iterations per epoch, so that with d_steps_per_g = 2 an epoch ends in the middle of a G D D cycle.  Run A trains
epochs 0-1 and writes checkpoint_2.pth; run B resumes from it (other initial weights, so the load shows) and trains to
epoch 6 with the linear decay from epoch 3.  Reconstruction: run A trains epochs 0-1 with a halving every 2 epochs,
run B resumes to epoch 5.  Search: five numbered checkpoints whose running-average generator carries its epoch in
fc.bias[0], scored by a stand-in FID with ties.

The checkpoints the reference wrote are kept in checkpoint_reference.npz as data (`encode`): a JSON manifest of the dict
(keys and their types, nesting, lists / tuples, Python scalars) plus one array per tensor.  `decode` rebuilds the same
dict, which a test saves with torch.save to get the file back."""
import json
import os

import numpy as np
import torch

import recon_step_common as RS
import wrapper_common as WC

GAN_ITERS, GAN_SEED_A, GAN_SEED_B, GAN_NOISE_A, GAN_NOISE_B = 4, 3, 11, 77, 78
GAN_EPOCHS_A, GAN_EPOCHS_B, GAN_DECAY_AFTER_B = 2, 6, 3
RECON_EPOCHS_A, RECON_EPOCHS_B, RECON_DECAY_EVERY, RECON_SEED_A, RECON_SEED_B = 2, 5, 2, 6, 16
SEARCH_FID = {100: 3.0, 40: 2.0, 20: 2.0, 10: 2.5, 5: 2.0}     # newest first: 40 is best, the ties at 20 and 5 do not replace it


def gan_args():
    a = WC.make_args(2, 512)
    a.d_steps_per_g, a.mesh_regularization, a.conditional_class, a.tensorboard = 2, 0.0001, True, False
    a.lr_g, a.lr_d, a.texture_only = 0.01, 0.04, False
    return a


def gan_inputs():
    """The batches of one epoch, as step's keyword arguments."""
    return [{k: v for k, v in WC.inputs(seed=50 + i, B=4).items() if k != "noise"} for i in range(GAN_ITERS)]


def gan_loader():
    """gan_inputs() as the reference's train_loader yields them."""
    return [{"texture": d["X_tex"], "texture_alpha": d["X_alpha"], "mesh": d["X_mesh"], "class": d["C"],
             "idx": torch.arange(4)} for d in gan_inputs()]


def recon_args():
    return RS.make_args(True, True)


def recon_batches():
    return [(X, s, t, r, idx.squeeze(-1)) for X, s, t, r, idx in RS.batches()]


def adam_state(opt):
    """{'<i>.<name>': tensor} of an optimiser's per-parameter state, i = the parameter's index in its group."""
    out = {}
    params = [p for g in opt.param_groups for p in g["params"]]
    for i, p in enumerate(params):
        for k, v in opt.state[p].items():
            out[f"{i}.{k}"] = torch.as_tensor(v).detach().cpu()
    return out


def write_search_checkpoints(directory):
    """checkpoint_<e>.pth for every epoch of SEARCH_FID, plus a checkpoint_latest.pth the glob must skip."""
    gi, _ = WC.build()
    for e in list(SEARCH_FID) + ["latest"]:
        G, avg = gi(), gi()
        with torch.no_grad():
            avg.fc.bias[0] = float(e) if e != "latest" else -1.0
            G.fc.bias[0] = -float(e) if e != "latest" else 1.0
        torch.save({"generator": G.state_dict(), "generator_running_avg": avg.state_dict(),
                    "epoch": e if e != "latest" else 0, "iteration": 0, "g_curve": [0], "d_fake_curve": [0],
                    "d_real_curve": [0], "flat_curve": [0]}, os.path.join(directory, f"checkpoint_{e}.pth"))


def search_fid(generator_running_avg):
    """The stand-in FID of the running-average generator a search checkpoint was loaded into."""
    return SEARCH_FID[int(round(float(generator_running_avg.fc.bias[0].detach())))]


def encode(obj, name, out):
    """A checkpoint dict -> out[name + '.manifest'] (JSON of its structure and Python values) and out[f'{name}.<i>'] (its
    tensors, in order)."""
    tensors = []

    def enc(x):
        if isinstance(x, torch.Tensor):
            tensors.append(x.detach().cpu())
            return {"tensor": len(tensors) - 1, "dtype": str(x.dtype)}
        if isinstance(x, dict):
            return {"dict": [[enc(k), enc(v)] for k, v in x.items()]}
        if isinstance(x, (list, tuple)):
            return {type(x).__name__: [enc(v) for v in x]}
        if x is None or isinstance(x, (bool, int, float, str)):
            return {"value": x}
        raise TypeError(f"{name}: cannot encode {type(x)}")
    out[name + ".manifest"] = np.array(json.dumps(enc(obj)))
    for i, t in enumerate(tensors):
        out[f"{name}.{i}"] = t.numpy().copy()


def decode(golden, name):
    """The dict `encode` stored under name (same keys, nesting, Python types, tensor dtypes and values)."""
    def dec(x):
        if "tensor" in x:
            t = torch.from_numpy(np.array(golden[f"{name}.{x['tensor']}"]))
            assert str(t.dtype) == x["dtype"], (name, t.dtype, x["dtype"])
            return t
        if "dict" in x:
            return {dec(k): dec(v) for k, v in x["dict"]}
        if "tuple" in x:
            return tuple(dec(v) for v in x["tuple"])
        if "list" in x:
            return [dec(v) for v in x["list"]]
        return x["value"]
    return dec(json.loads(str(golden[name + ".manifest"])))
