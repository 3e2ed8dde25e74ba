"""`DataParallelWithCallback` of the reference (sync_batchnorm/replicate.py:50-67) exists to run SyncBN under
single-process nn.DataParallel.  The design is one process per GPU (torchrun + NCCL), where
SynchronizedBatchNorm2d synchronises through torch.distributed by itself; this wrapper therefore only keeps the
import and call surface of main.py:149,530-548 alive: it behaves like the wrapped module (`.module`, forward)."""
import torch.nn as nn


class DataParallelWithCallback(nn.Module):
    def __init__(self, module, device_ids=None, output_device=None, dim=0):
        super().__init__()
        if device_ids is not None and len(device_ids) > 1:
            raise RuntimeError("single-process multi-GPU DataParallel is not part of the design: launch one "
                               "process per GPU with torchrun (see gan_training.py / INTEGRATION.md)")
        self.module = module

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)


def patch_replication_callback(data_parallel):
    return data_parallel
