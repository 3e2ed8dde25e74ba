"""What main.py and run_reconstruction.py share: one process per GPU under torchrun, the log file, the Inception check,
the per-iteration log lines and scalars (formatted at the end of an epoch from values read in one synchronisation), and
the TensorBoard image grids (built on the device, copied to the host once each)."""
import os
import shutil
import sys

import torch
import torch.distributed as dist

from sample_export import grid_shape, place_tiles


# ------------------------------------------------------------------------------------------------ processes and devices
def init_devices(gpu_ids, script, argv):
    """-> (rank, world, device).  Under torchrun (WORLD_SIZE > 1) every process takes GPU LOCAL_RANK and joins an NCCL
    group; otherwise --gpu_ids must name one GPU.  A list of several ids outside torchrun exits with the command that runs
    one process per GPU (the drivers never spawn processes)."""
    ids = [int(x) for x in gpu_ids.split(',')]
    world = int(os.environ.get('WORLD_SIZE', '1'))
    if world == 1 and len(ids) > 1:
        raise SystemExit(f'error: --gpu_ids {gpu_ids} names {len(ids)} GPUs; this program runs one process per GPU. '
                         f'Start it with\n  CUDA_VISIBLE_DEVICES={gpu_ids} torchrun --nproc-per-node {len(ids)} {script} '
                         + ' '.join(argv))
    if world > 1:
        device = torch.device('cuda', int(os.environ['LOCAL_RANK']))
        torch.cuda.set_device(device)
        dist.init_process_group('nccl', device_id=device)
        return dist.get_rank(), world, device
    device = torch.device('cuda', ids[0])
    torch.cuda.set_device(device)
    return 0, 1, device


def shutdown(world):
    """Leave the process group once every rank is done (rank 0 may still be writing an export)."""
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def per_rank_batch(batch_size, world):
    """--batch_size is the global batch, split evenly over the ranks as DataParallel splits it."""
    if batch_size % world:
        raise SystemExit(f'error: --batch_size {batch_size} is not divisible by the {world} processes')
    return batch_size // world


def load_inception():
    """The Inception network of the FID scores, from $B3D_INCEPTION_WEIGHTS or the torch hub cache (never downloaded),
    loaded before any other work so that a missing file stops the run at once."""
    from utils.fid import init_inception
    try:
        return init_inception()
    except FileNotFoundError as e:
        raise SystemExit(f'error: {e}')


def command_line(script, argv):
    """The first line of log.txt: the command as sys.argv gives it."""
    return ' '.join(sys.argv if argv is None else [script] + list(argv))


class Log:
    """log(text): print, and append to log.txt when a path is given (line-buffered); only rank 0 writes."""

    def __init__(self, path=None, append=False, first_line=None, rank=0):
        self.rank, self.file = rank, None
        if path is not None and rank == 0:
            self.file = open(path, 'a' if append else 'w', buffering=1)
            print(first_line, file=self.file)

    def __call__(self, text):
        if self.rank:
            return
        if self.file is not None:
            print(text, file=self.file)
        print(text)

    def close(self):
        if self.file is not None:
            self.file.close()


def summary_writer(log_dir, clear, rank=0):
    """torch.utils.tensorboard.SummaryWriter on rank 0 (None elsewhere); clear deletes earlier events first."""
    if rank:
        return None
    from torch.utils.tensorboard import SummaryWriter
    if clear:
        shutil.rmtree(log_dir, ignore_errors=True)
    return SummaryWriter(log_dir)


# ------------------------------------------------------------------------------------------------ log lines
GAN_LINE = '[{}] epoch {}, {}/{}, g_loss {:.5f} d_fake_loss {:.5f} d_real_loss {:.5f} flat {:.5f}'
RECON_LINE = '[{}] epoch {}, {}/{}, recon_loss {:.5f} flat_loss {:.5f} total {:.5f} iou {:.5f}'
TIME_LINE = 'Time per epoch: {:.3f} s'
TEST_LINE = '[TEST] recon_loss {:.5f}, flat_loss {:.5f}, mIoU {:.5f}, N {}'


def gan_epoch_records(it0, epoch, n_iters, d_steps_per_g, loss, curves, lengths, use_mesh):
    """One epoch of main.py's loop (:691-736) replayed from the curves GANTrainer.train_epoch extended: curves (g, d_fake,
    d_real, flat) after the epoch, lengths their lengths before it.  -> (log lines: the line of every iteration whose
    global number is a multiple of 10, with the curves' last values at that iteration; scalars: (tag, value, step) in
    the order the reference writes them)."""
    g, d_fake, d_real, flat = curves
    ng, nd, nf = lengths[0], lengths[1], lengths[3]
    lines, scalars = [], []
    for i in range(n_iters):
        k = it0 + i
        if k % (1 + d_steps_per_g) == 0:
            ng += 1
            scalars.append((f'gan_{loss}/g', g[ng - 1], k))
            if use_mesh:
                nf += 1
                scalars.append(('flat', flat[nf - 1], k))
        else:
            nd += 1
            scalars.append((f'gan_{loss}/d_fake_loss', d_fake[nd - 1], k))
            scalars.append((f'gan_{loss}/d_real_loss', d_real[nd - 1], k))
        if k % 10 == 0:
            lines.append(GAN_LINE.format(k, epoch, i, n_iters, g[ng - 1], d_fake[nd - 1], d_real[nd - 1], flat[nf - 1]))
    return lines, scalars


def recon_epoch_records(it0, epoch, n_iters, loss, values):
    """One epoch of run_reconstruction.py's loop (:448-458) from ReconTrainer.train_epoch's per-step (loss, recon, flat,
    miou) values, read to the host once.  -> (log lines, scalars (tag, value, step))."""
    lines, scalars = [], []
    for i, (total, recon, flat, miou) in enumerate(values):
        k = it0 + i
        if k % 10 == 0:
            lines.append(RECON_LINE.format(k, epoch, i, n_iters, recon, flat, total, miou))
        scalars += [(f'{loss}/train', recon, k), ('flat/train', flat, k), ('iou/train', miou, k)]
    return lines, scalars


def fid_lines(scores):
    """main.py:348-376's lines from FIDEvaluator.evaluate's scores."""
    lines = ['FID (training set): {:.02f}'.format(scores['fid'])]
    if 'fid_texture_only' in scores:
        lines.append('Texture-only FID (training set): {:.02f}'.format(scores['fid_texture_only']))
        lines.append('Mesh-only FID (training set): {:.02f}'.format(scores['fid_mesh_only']))
    if 'fid_val' in scores:
        lines.append('FID (validation set): {:.02f}'.format(scores['fid_val']))
        if 'fid_texture_only_val' in scores:
            lines.append('Texture-only FID (validation set): {:.02f}'.format(scores['fid_texture_only_val']))
            lines.append('Mesh-only FID (validation set): {:.02f}'.format(scores['fid_mesh_only_val']))
    return lines


def test_line(stats):
    return TEST_LINE.format(stats['recon_loss'], stats['flat_loss'], stats['miou'], stats['N'])


def write_scalars(writer, scalars):
    if writer is not None:
        for tag, value, step in scalars:
            writer.add_scalar(tag, value, step)


# ------------------------------------------------------------------------------------------------ image grids
@torch.no_grad()
def make_grid(x, nrow, padding=2):
    """torchvision.utils.make_grid(x, nrow, padding) for [N,3,H,W] tensors (pad value 0), on x's device -> [3, H', W']."""
    if x.shape[0] == 1:
        return x[0]
    shape, cols = grid_shape(x.shape[0], x.shape[2], x.shape[3], nrow, padding)
    grid = x.new_zeros(shape)
    place_tiles(grid, cols, 0, x.permute(0, 2, 3, 1), padding)
    return grid.permute(2, 0, 1)


@torch.no_grad()
def to_grid_tex(x):
    """main.py:656-658: textures in [-1, 1] -> (x + 1) / 2 in a grid of four columns."""
    return make_grid((x[:, :3] + 1) / 2, nrow=4)


@torch.no_grad()
def to_grid_mesh(x):
    """main.py:660-666: every channel of every mesh map scaled to [0, 1] by its own minimum and maximum."""
    x = x[:, :3]
    minv = x.amin(dim=(2, 3), keepdim=True)
    maxv = x.amax(dim=(2, 3), keepdim=True)
    return make_grid((x - minv) / (maxv - minv), nrow=4)


@torch.no_grad()
def to_grid(x):
    """run_reconstruction.py:234-235: the first 16 images of [-1, 1] RGB(A) batches, four columns."""
    return make_grid((x[:16, :3] + 1) / 2, nrow=4)


def add_image(writer, tag, grid, step):
    """One device-to-host copy per grid."""
    writer.add_image(tag, grid.float().cpu().numpy(), step)


def merge_samples(parts, samples):
    """The visualisation samples each rank found in its shard ({'index': [k], field: [k, ...]}, rank order) as one set
    in the order `samples` lists the dataset indices."""
    merged = {k: torch.cat([p[k] for p in parts if k in p]) for k in set().union(*parts)}
    pos = {int(i): j for j, i in enumerate(samples)}
    order = torch.argsort(torch.tensor([pos[int(i)] for i in merged['index']]))
    return {k: v[order] for k, v in merged.items()}


def gather_to_rank0(obj, world):
    """Every rank's obj (host tensors / arrays) as a list in rank order on rank 0 ([obj] without torch.distributed)."""
    if world == 1:
        return [obj]
    out = [None] * world if dist.get_rank() == 0 else None
    dist.gather_object(obj, out, dst=0)
    return out
