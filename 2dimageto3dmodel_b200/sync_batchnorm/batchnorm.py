"""SynchronizedBatchNorm{1,2,3}d with the reference's state-dict layout (they extend _BatchNorm:
running_mean / running_var / num_batches_tracked, optional weight / bias).

Single process (world size 1) or eval mode: F.batch_norm, exactly like the reference's non-parallel branch
(batchnorm.py:69-73).  Under torch.distributed with world size > 1 and training: the reference's parallel
formulas (batchnorm.py:133-150) — mean = S/n, var = (SS - S*mean)/n, inv_std = clamp(var, eps)^-1/2, running
variance unbiased — with S, SS summed over all ranks by one all-reduce (and one in the backward)."""
import torch
import torch.distributed as dist
import torch.nn.functional as F
from torch.nn.modules.batchnorm import _BatchNorm


def _world():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


class _SyncStats(torch.autograd.Function):
    """x [B,C,*] -> (x - mean) * inv_std with statistics over the global batch."""

    @staticmethod
    def forward(ctx, x, eps, group):
        C = x.shape[1]
        red = [0] + list(range(2, x.dim()))
        stats = torch.stack((x.sum(dim=red), (x * x).sum(dim=red)))            # [2, C]
        dist.all_reduce(stats, group=group)
        n = x.numel() // C * dist.get_world_size(group)
        mean = stats[0] / n
        var = (stats[1] - stats[0] * mean) / n
        inv_std = var.clamp(min=eps) ** -0.5
        shape = [1, C] + [1] * (x.dim() - 2)
        xhat = (x - mean.view(shape)) * inv_std.view(shape)
        ctx.save_for_backward(xhat, inv_std, var >= eps)
        ctx.group, ctx.n = group, n
        ctx.mark_non_differentiable(mean, var)
        return xhat, mean, var

    @staticmethod
    def backward(ctx, g, _gm, _gv):
        xhat, inv_std, unclamped = ctx.saved_tensors
        C = xhat.shape[1]
        red = [0] + list(range(2, xhat.dim()))
        sums = torch.stack((g.sum(dim=red), (g * xhat).sum(dim=red)))
        dist.all_reduce(sums, group=ctx.group)
        shape = [1, C] + [1] * (xhat.dim() - 2)
        # d clamp(var, eps) / d var = 0 where the variance is clamped: no xhat coupling term in those channels
        gx = (g - sums[0].view(shape) / ctx.n - xhat * (sums[1] * unclamped / ctx.n).view(shape)) * inv_std.view(shape)
        return gx, None, None


class _SynchronizedBatchNorm(_BatchNorm):
    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True,
                 process_group=None):
        super().__init__(num_features, eps=eps, momentum=momentum, affine=affine,
                         track_running_stats=track_running_stats)
        self.process_group = process_group

    def _check_input_dim(self, input):
        pass

    def forward(self, input):
        if not (self.training and _world() > 1):
            return F.batch_norm(input, self.running_mean, self.running_var, self.weight, self.bias, self.training,
                                self.momentum, self.eps)
        xhat, mean, var = _SyncStats.apply(input, self.eps, self.process_group)
        if self.track_running_stats:
            n = input.numel() // input.shape[1] * _world()
            with torch.no_grad():
                self.running_mean.mul_(1 - self.momentum).add_(mean, alpha=self.momentum)
                self.running_var.mul_(1 - self.momentum).add_(var * (n / max(n - 1, 1)), alpha=self.momentum)
                self.num_batches_tracked += 1
        if self.affine:
            shape = [1, -1] + [1] * (input.dim() - 2)
            xhat = xhat * self.weight.view(shape) + self.bias.view(shape)
        return xhat


class SynchronizedBatchNorm1d(_SynchronizedBatchNorm):
    pass


class SynchronizedBatchNorm2d(_SynchronizedBatchNorm):
    pass


class SynchronizedBatchNorm3d(_SynchronizedBatchNorm):
    pass


def convert_model(module):
    """nn.BatchNormNd -> SynchronizedBatchNormNd, recursively (same parameters and buffers)."""
    mapping = {torch.nn.BatchNorm1d: SynchronizedBatchNorm1d, torch.nn.BatchNorm2d: SynchronizedBatchNorm2d,
               torch.nn.BatchNorm3d: SynchronizedBatchNorm3d}
    for src, dst in mapping.items():
        if isinstance(module, src):
            new = dst(module.num_features, module.eps, module.momentum, module.affine, module.track_running_stats)
            new.load_state_dict(module.state_dict())
            return new
    for name, child in module.named_children():
        module.add_module(name, convert_model(child))
    return module
