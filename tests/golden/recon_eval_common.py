"""Shared by make_golden_recon_eval.py (reference side) and the validation-pass tests (drop-in side): the seeded changes
that make the evaluation goldens depend on what a validation pass reads — batch-norm running statistics (eval mode uses
them instead of batch statistics) and DatasetParams away from their initial values (the pass poses with their dataset
mean) — plus the stand-in validation batches and the options evaluated."""
import torch

# (tag, optimize_deltas, optimize_z0); the reference cannot run with neither (transform_vertices :251)
POSES = (("deltas", True, False), ("full", True, True), ("z0", False, True))
CRITERIA = ("mse", "l1")
MULTIVIEW_IDX = 1


def set_running_stats(net, seed=55):
    """running_mean ~ N(0, 0.2), running_var ~ U(0.5, 2) for every batch norm, in sorted buffer-name order."""
    g = torch.Generator().manual_seed(seed)
    sd = net.state_dict()
    with torch.no_grad():
        for k in sorted(k for k in sd if k.endswith(".running_mean")):
            mean, var = sd[k], sd[k[:-len("running_mean")] + "running_var"]
            mean.copy_(torch.randn(mean.shape, generator=g) * 0.2)
            var.copy_(0.5 + 1.5 * torch.rand(var.shape, generator=g))
    return net


def perturb_dataset_params(dp, seed=8):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name in ("ds_translation", "ds_scale", "ds_z0"):
            p = getattr(dp, name, None)
            if p is not None:
                p.add_((torch.randn(p.shape, generator=g) * 0.1).to(p.device))
    return dp


def eval_batches():
    """Three stand-in batches of 4 (recon_step_common's scene) -> N = 12."""
    import recon_step_common as RS
    return RS.batches(n=3, B=4, seed=29)
