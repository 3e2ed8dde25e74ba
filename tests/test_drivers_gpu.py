"""The command-line drivers end to end on one synthetic CUB tree: reconstruction training, resume, evaluation and
pseudo-ground-truth export with run_reconstruction.py, then GAN training, best-epoch evaluation and sample export with
main.py on the exported cache, each step a subprocess run from the tree as a user runs it.  Then the host
synchronisations of an epoch, counted in-process, do not grow with its number of iterations."""
import os
import re
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

from conftest import PKG, ROOT

pytestmark = pytest.mark.gpu
N_TRAIN, N_VAL = 24, 8


@pytest.fixture(scope='module')
def tree(tmp_path_factory):
    from fid_common import randomize_inception
    from tools.time_recon_data import write_cub_like_tree
    from tools.uvsphere import write_uvsphere_obj
    from utils.fid import init_inception
    root = str(tmp_path_factory.mktemp('drivers'))
    write_cub_like_tree(root, N_VAL, seed=5, split='testval')
    write_cub_like_tree(root, N_TRAIN, seed=4, split='train')
    labels = os.path.join(root, 'datasets', 'cub', 'CUB_200_2011')
    names = [f'001.Synthetic/Bird_{i:05d}.jpg' for i in range(N_TRAIN)]
    with open(os.path.join(labels, 'images.txt'), 'w') as f:
        f.write(''.join(f'{i + 1} {p}\n' for i, p in enumerate(names)))
    with open(os.path.join(labels, 'image_class_labels.txt'), 'w') as f:
        f.write(''.join(f'{i + 1} {i % 3 + 1}\n' for i in range(N_TRAIN)))
    os.makedirs(os.path.join(root, 'mesh_templates'))
    write_uvsphere_obj(os.path.join(root, 'mesh_templates', 'uvsphere_16rings.obj'), rings=16)
    inc = os.path.join(root, 'inception.pth')
    torch.save(randomize_inception(init_inception(weights=None), 3).state_dict(), inc)
    return root


def run(tree, script, *argv):
    env = dict(os.environ, B3D_INCEPTION_WEIGHTS=os.path.join(tree, 'inception.pth'))
    r = subprocess.run([sys.executable, os.path.join(PKG, script), *argv], cwd=tree, env=env, capture_output=True,
                       text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def events(logdir):
    ea = pytest.importorskip('tensorboard.backend.event_processing.event_accumulator')
    acc = ea.EventAccumulator(logdir, size_guidance={ea.SCALARS: 0, ea.IMAGES: 0})
    acc.Reload()
    return acc.Tags()


RECON = ('--name', 't', '--dataset', 'cub', '--batch_size', '8', '--evaluate_freq', '1', '--save_freq', '1')


def test_1_recon_training_writes_checkpoints_log_and_summaries(tree):
    run(tree, 'run_reconstruction.py', *RECON, '--epochs', '2', '--tensorboard', '--image_freq', '1')
    d = os.path.join(tree, 'checkpoints_recon', 't')
    assert os.path.exists(os.path.join(d, 'checkpoint_latest.pth'))
    log = open(os.path.join(d, 'log.txt')).read().splitlines()
    assert log[0].endswith('run_reconstruction.py ' + ' '.join(RECON) + ' --epochs 2 --tensorboard --image_freq 1')
    assert re.fullmatch(r'\[0\] epoch 0, 0/3, recon_loss \d+\.\d{5} flat_loss \d+\.\d{5} total \d+\.\d{5} iou \d\.\d{5}', log[1])
    assert sum(line.startswith('Time per epoch: ') for line in log) == 2
    assert sum(line.startswith('[TEST] recon_loss ') for line in log) == 2
    tags = events(os.path.join(tree, 'tensorboard_recon', 't'))
    assert {'mse/train', 'flat/train', 'iou/train', 'mse/val', 'flat/val', 'iou/val'} <= set(tags['scalars'])
    assert {'image_train/real', 'image_train/fake', 'image_val/real', 'image_val/fake', 'image_val/render'} <= set(tags['images'])


def test_2_recon_resume_appends(tree):
    out = run(tree, 'run_reconstruction.py', *RECON, '--epochs', '3', '--continue_train')
    assert 'Resuming from epoch 2' in out
    log = open(os.path.join(tree, 'checkpoints_recon', 't', 'log.txt')).read().splitlines()
    assert sum('run_reconstruction.py --name t' in line for line in log) == 2
    assert sum(line.startswith('Time per epoch: ') for line in log) == 3
    assert torch.load(os.path.join(tree, 'checkpoints_recon', 't', 'checkpoint_latest.pth'))['epoch'] == 3


def test_3_recon_evaluate_prints_the_test_line_of_recon_trainer(tree):
    import command_line as cl
    import run_reconstruction as rr
    from cmr_data.cub import CUBDataset
    from reconstruction_training import ReconTrainer
    from rendering.mesh_template import MeshTemplate
    out = run(tree, 'run_reconstruction.py', '--name', 't', '--dataset', 'cub', '--batch_size', '8', '--evaluate')
    args = rr.build_parser().parse_args(['--name', 't', '--dataset', 'cub'])
    tpl = MeshTemplate(os.path.join(tree, 'mesh_templates', 'uvsphere_16rings.obj'), device='cuda')
    rec = ReconTrainer(args, tpl, N_TRAIN)
    rec.load_checkpoint(os.path.join(tree, 'checkpoints_recon', 't', 'checkpoint_latest.pth'), 'evaluate')
    val = CUBDataset('testval', False, 256, root=tree).to_device('cuda')
    assert cl.test_line(rec.evaluate(val.eval_batches(8))) in out.splitlines()


def test_4_pseudogt_export(tree):
    run(tree, 'run_reconstruction.py', '--name', 't', '--dataset', 'cub', '--batch_size', '8', '--generate_pseudogt',
        '--pseudogt_resolution', '256')
    cache = os.path.join(tree, 'cache', 'cub')
    assert len(os.listdir(os.path.join(cache, 'pseudogt_256x256'))) == N_TRAIN
    for f in ('poses_metadata.npz', 'precomputed_fid_299x299_train.npz', 'precomputed_fid_299x299_testval.npz'):
        assert os.path.exists(os.path.join(cache, f)), f


GAN = ('--weights', 'g', '--dataset', 'cub', '--texture_resolution', '256')


def test_5_gan_training(tree):
    run(tree, 'main.py', *GAN, '--batch_size', '4', '--epochs', '2', '--evaluate_freq', '1', '--save_freq', '1',
        '--checkpoint_freq', '1', '--tensorboard')
    d = os.path.join(tree, 'gan_weights', 'g')
    for f in ('checkpoint_latest.pth', 'checkpoint_1.pth', 'checkpoint_2.pth'):
        assert os.path.exists(os.path.join(d, f)), f
    log = open(os.path.join(d, 'log.txt')).read().splitlines()
    assert 'main.py --weights g' in log[0]
    assert re.fullmatch(r'\[0\] epoch 0, 0/6, g_loss -?\d+\.\d{5} d_fake_loss 0\.00000 d_real_loss 0\.00000 flat \d+\.\d{5}',
                        log[1]), log[1]
    for head in ('FID (training set): ', 'Texture-only FID (training set): ', 'Mesh-only FID (training set): ',
                 'FID (validation set): '):
        assert sum(line.startswith(head) for line in log) == 2, head
    tags = events(os.path.join(tree, 'tensorboard_gan', 'g'))
    assert {'gan_hinge/g', 'gan_hinge/d_fake_loss', 'gan_hinge/d_real_loss', 'flat', 'fid/combined', 'fid/combined_val',
            'fid/texture_only', 'fid/mesh_only'} <= set(tags['scalars'])
    assert {'image/real_tex', 'image/fake_tex', 'image/fake_mesh', 'render/fake', 'render/fake_texture',
            'render/fake_mesh', 'render/real'} <= set(tags['images'])


def test_6_gan_evaluate_best(tree, monkeypatch):
    """The driver's search picks, scores and prints what select_best_checkpoint gives in this process on the same files."""
    import command_line as cl
    import main
    from fid_evaluation import select_best_checkpoint
    from gan_training import GANTrainer
    from rendering.mesh_template import MeshTemplate
    from utils.fid import init_inception
    out = run(tree, 'main.py', *GAN, '--batch_size', '4', '--evaluate', '--which_epoch', 'best').splitlines()
    args = main.build_parser().parse_args(list(GAN) + ['--batch_size', '4', '--evaluate'])
    ds = main.make_dataset(args, root=tree)
    main.derive_settings(args, ds)
    ds.to_device('cuda')
    tpl = MeshTemplate(os.path.join(tree, args.mesh_path), is_symmetric=args.symmetric_g, device='cuda')
    gan = GANTrainer(args, mesh_template=tpl)
    ev = main.make_evaluator(args, ds, gan.trainer.generator_running_avg, tpl,
                             init_inception(os.path.join(tree, 'inception.pth')), 'cuda')
    monkeypatch.chdir(tree)                       # the driver globs gan_weights/g relative to its working directory
    best = select_best_checkpoint(gan, ev, os.path.join('gan_weights', 'g'), main.EvalBatches(ds, 4, 0, 1), seed=1234)
    assert sorted(best['fast_fid']) == [1, 2]
    assert f'--- Running final evaluation using {best["best_path"]} ---' in out
    i = out.index('--- Running final evaluation using ' + best['best_path'] + ' ---')
    assert out[i + 1:i + 1 + len(cl.fid_lines(best['scores']))] == cl.fid_lines(best['scores'])
    # 'Best FID so far' prints the full float: compare its path, and every other line exactly
    got, want = out[out.index('Enumerating checkpoints:'):i + 1], main.search_lines(best)
    assert [best_path_only(x) for x in got] == [best_path_only(x) for x in want]


def best_path_only(line):
    return line.split(' at ')[-1] if line.startswith('Best FID so far: ') else line


def test_7_gan_save_results(tree):
    run(tree, 'main.py', *GAN, '--batch_size', '4', '--save_results')
    d = os.path.join(tree, 'results', 'g')
    for i in range(4):
        for ext in ('obj', 'mtl', 'png'):
            assert os.path.getsize(os.path.join(d, f'mesh_{i}.{ext}')) > 0
    v = sum(1 for line in open(os.path.join(d, 'mesh_0.obj')) if line.startswith('v '))
    from rendering.mesh_template import MeshTemplate
    assert v == MeshTemplate(os.path.join(tree, 'mesh_templates', 'uvsphere_16rings.obj')).mesh.vertices.shape[0]
    from PIL import Image
    assert Image.open(os.path.join(tree, 'results', 'g.png')).size == (4 * 256, 256)


def sync_count(fn):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum('synchroniz' in str(x.message) for x in w)


@pytest.mark.parametrize('script', ['main', 'run_reconstruction'])
def test_8_no_synchronisation_per_iteration(tree, script, monkeypatch):
    """24 samples in batches of 6 and of 2: 4 and 12 iterations per epoch, the same synchronisations per epoch (those of
    a 3-epoch run less those of a 1-epoch run, so that the one-time set-up cancels).  The caching allocator may free and
    re-allocate once as the larger batches' memory grows, which counts as one synchronisation; one per iteration would
    add 8 per epoch.  Runs on the caches and checkpoints the steps above wrote."""
    import importlib
    mod = importlib.import_module(script)
    monkeypatch.chdir(tree)
    monkeypatch.setenv('B3D_INCEPTION_WEIGHTS', os.path.join(tree, 'inception.pth'))
    per_epoch = []
    for b in (6, 2):
        c = {}
        for e in (1, 3):
            if script == 'main':
                argv = ['--weights', f's{b}_{e}', '--dataset', 'cub', '--texture_resolution', '256', '--evaluate_freq', '100']
            else:
                argv = ['--name', f's{b}_{e}', '--dataset', 'cub']
            c[e] = sync_count(lambda: mod.main(argv + ['--batch_size', str(b), '--epochs', str(e), '--save_freq', '1']))
        per_epoch.append((c[3] - c[1]) / 2)
    assert abs(per_epoch[0] - per_epoch[1]) <= 1, per_epoch
