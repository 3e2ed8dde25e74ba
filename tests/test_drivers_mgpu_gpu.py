"""The drivers' multi-process paths under `torchrun --nproc-per-node 2`, on the synthetic CUB tree of test_drivers_gpu.py:
reconstruction training with validation images, pseudo-ground-truth export (rank 0), GAN training with FID and image
summaries, the best-epoch search and the sample export (rank 0).  Every run must finish on both ranks, only rank 0 may
write the log, the checkpoints and the events, and the image grids gathered from both ranks' shards must hold every
visualisation sample.  The losses are not compared with a one-GPU run: each rank draws its generator noise and its
mirror flips from its own stream, and the ranks' sample orders come from DistributedSampler (INTEGRATION.md
"Command line").  Skipped on a machine with fewer than two GPUs."""
import os
import subprocess
import sys

import pytest
import torch

from conftest import PKG
from test_drivers_gpu import N_TRAIN, events, tree  # noqa: F401  (the module-scoped synthetic tree)

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")]


def torchrun(tree, script, *argv):
    env = dict(os.environ, B3D_INCEPTION_WEIGHTS=os.path.join(tree, 'inception.pth'), TORCH_NCCL_ASYNC_ERROR_HANDLING='0')
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2', '--master-addr', '127.0.0.1',
           '--master-port', str(29500 + os.getpid() % 400), os.path.join(PKG, script), *argv]
    r = subprocess.run(cmd, cwd=tree, env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def image_size(logdir, tag):
    from tensorboard.backend.event_processing import event_accumulator as ea
    acc = ea.EventAccumulator(logdir, size_guidance={ea.IMAGES: 0})
    acc.Reload()
    im = acc.Images(tag)[-1]
    return im.width, im.height


def count(lines, head):
    return sum(line.startswith(head) for line in lines)


def test_1_recon_training_on_two_ranks(tree):
    torchrun(tree, 'run_reconstruction.py', '--name', 'm', '--dataset', 'cub', '--batch_size', '8', '--epochs', '2',
             '--evaluate_freq', '1', '--save_freq', '1', '--tensorboard', '--image_freq', '1')
    d = os.path.join(tree, 'checkpoints_recon', 'm')
    log = open(os.path.join(d, 'log.txt')).read().splitlines()
    assert count(log, '[0] epoch 0, 0/3,') == 1 and count(log, 'Time per epoch') == 2 and count(log, '[TEST] ') == 2
    assert torch.load(os.path.join(d, 'checkpoint_latest.pth'))['iteration'] == 6
    assert sorted(os.listdir(os.path.join(tree, 'tensorboard_recon'))) == ['m']
    assert len(os.listdir(os.path.join(tree, 'tensorboard_recon', 'm'))) == 1          # one event file: rank 0's
    # debug ids 0 and 1 of the 8 validation images: two 256^2 tiles, four columns, 2-pixel padding
    assert image_size(os.path.join(tree, 'tensorboard_recon', 'm'), 'image_val/real') == (2 * 258 + 2, 260)


def test_2_pseudogt_export_on_rank_0(tree):
    out = torchrun(tree, 'run_reconstruction.py', '--name', 'm', '--dataset', 'cub', '--batch_size', '8',
                   '--generate_pseudogt', '--pseudogt_resolution', '256')
    assert out.count('Done.') == 1
    assert len(os.listdir(os.path.join(tree, 'cache', 'cub', 'pseudogt_256x256'))) == N_TRAIN


def test_3_gan_training_on_two_ranks(tree):
    torchrun(tree, 'main.py', '--weights', 'm', '--dataset', 'cub', '--texture_resolution', '256', '--batch_size', '4',
             '--epochs', '2', '--evaluate_freq', '1', '--save_freq', '1', '--checkpoint_freq', '1', '--tensorboard')
    d = os.path.join(tree, 'gan_weights', 'm')
    log = open(os.path.join(d, 'log.txt')).read().splitlines()
    assert count(log, '[0] epoch 0, 0/6,') == 1 and count(log, 'Time per epoch') == 2
    assert count(log, 'FID (training set): ') == 2 and count(log, 'FID (validation set): ') == 2
    chk = torch.load(os.path.join(d, 'checkpoint_2.pth'))
    assert chk['epoch'] == 2 and chk['iteration'] == 12
    logdir = os.path.join(tree, 'tensorboard_gan', 'm')
    assert len(os.listdir(logdir)) == 1
    # the last batch's 4 indices, 2 from each rank's training shard, found across both evaluation shards: 4 tiles
    assert image_size(logdir, 'render/fake') == (4 * 301 + 2, 303)
    assert image_size(logdir, 'image/fake_tex') == (4 * 258 + 2, 260)


def test_4_gan_best_epoch_search_on_two_ranks(tree):
    out = torchrun(tree, 'main.py', '--weights', 'm', '--dataset', 'cub', '--texture_resolution', '256', '--batch_size', '4',
                   '--evaluate', '--which_epoch', 'best').splitlines()
    assert count(out, 'Enumerating checkpoints:') == 1 and count(out, '--- Running final evaluation using ') == 1


def test_5_sample_export_on_rank_0(tree):
    out = torchrun(tree, 'main.py', '--weights', 'm', '--dataset', 'cub', '--texture_resolution', '256', '--batch_size', '4',
                   '--save_results')
    assert out.count('successfully done') == 1
    assert sorted(os.listdir(os.path.join(tree, 'results', 'm'))) == sorted(
        f'mesh_{i}.{e}' for i in range(4) for e in ('obj', 'mtl', 'png'))
