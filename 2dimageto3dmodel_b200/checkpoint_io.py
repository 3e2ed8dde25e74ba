"""Checkpoint files in the reference's format (main.py:749-770, run_reconstruction.py:472-481): `torch.save` dicts of state
dicts, counters and `vars(args)`, shared by `GANTrainer` and `ReconTrainer`.

The optimiser state is written the way a plain `optim.Adam` (the reference's) writes it, whatever implementation runs here:
`step` as a CPU fp32 tensor and the plain implementation flags (`foreach` / `fused` None, `capturable` False).  Loading puts
this trainer's own flags back and moves `step` where its Adam keeps it (on the device for the fused / capturable forms), so a
file goes both ways between the reference and the fused CUDA Adams.  `step` stored as a Python number, as torch < 1.12
wrote it, loads too.

Under torch.distributed rank 0 writes and every rank waits at a barrier; every rank reads the same file onto its own
device."""
import torch
import torch.distributed as dist

# the flags that select an Adam implementation, and their values in a plain optim.Adam(params, lr, betas)
_PLAIN_ADAM_FLAGS = dict(foreach=None, fused=None, capturable=False)


def _distributed():
    return dist.is_available() and dist.is_initialized()


def optimizer_state_dict(opt):
    """opt.state_dict() in the form a plain Adam writes it."""
    sd = opt.state_dict()
    state = {}
    for k, st in sd["state"].items():
        st = dict(st)
        if "step" in st:
            st["step"] = st["step"].detach().to("cpu", torch.float32, copy=True)
        state[k] = st
    groups = [{**g, **_PLAIN_ADAM_FLAGS} for g in sd["param_groups"]]
    return {"state": state, "param_groups": groups}


def load_optimizer_state_dict(opt, sd):
    """opt.load_state_dict(sd), keeping opt's own implementation flags; `step` goes to the parameter's device when the
    implementation reads it there (fused / capturable), else to the host."""
    flags = [{k: g[k] for k in _PLAIN_ADAM_FLAGS} for g in opt.param_groups]
    opt.load_state_dict(sd)               # a numeric step becomes a tensor here (Adam.__setstate__)
    for g, f in zip(opt.param_groups, flags):
        g.update(f)
        on_device = g["fused"] or g["capturable"]
        for p in g["params"]:
            st = opt.state.get(p)
            if st and "step" in st:
                st["step"] = st["step"].to(p.device if on_device else "cpu", torch.float32)


def save(obj, path):
    """torch.save on rank 0 (every process without torch.distributed); ends with a barrier under torch.distributed."""
    if not _distributed() or dist.get_rank() == 0:
        torch.save(obj, path)
    if _distributed():
        dist.barrier()


def load(path, device):
    return torch.load(path, map_location=device)
