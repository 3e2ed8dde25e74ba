"""main.py's epoch loop against GANTrainer.train_epoch called directly, on the same device batches at cfg3's size
(conditional CUB, B 32, 256^2 textures, two discriminators), alternated in one process:

    python tools/time_drivers.py [--iters 100] [--rounds 3] [--epochs 3]

A synthetic pseudo-ground-truth cache of iters * 32 records is written to a temporary directory.  Each round runs the
driver (`main.main`) for --epochs epochs and reads its 'Time per epoch' lines, then the same number of epochs of
train_epoch on the driver's batches with the same host clock; the first epoch of each run is warm-up.  Prints the card,
its power limit and both rates (iterations per second) as one JSON line.  CUDA only."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, '2dimageto3dmodel_b200'), ROOT]


def write_tree(root, n, R=256):
    from tools.uvsphere import write_uvsphere_obj
    g = torch.Generator().manual_seed(0)
    cache = os.path.join(root, 'cache', 'cub')
    pgt = os.path.join(cache, f'pseudogt_{R}x{R}')
    os.makedirs(pgt)
    names = [f'001.Synthetic/Bird_{i:05d}.jpg' for i in range(n)]
    np.savez(os.path.join(cache, 'poses_metadata'), data={
        'scale': 0.5 + torch.rand(n, 1, generator=g), 'translation': torch.randn(n, 3, generator=g) * 0.1,
        'rotation': torch.nn.functional.normalize(torch.randn(n, 4, generator=g), dim=1), 'path': names})
    tex = (torch.rand(3, R, R, generator=g) * 2 - 1).half()
    alpha = (torch.rand(1, R, R, generator=g) > 0.3).half()
    for i in range(n):
        np.savez(os.path.join(pgt, f'{i}'), data={'texture': tex, 'texture_alpha': alpha,
                                                  'mesh': torch.randn(3, 32, 32, generator=g) * 0.05})
    labels = os.path.join(root, 'datasets', 'cub', 'CUB_200_2011')
    os.makedirs(labels)
    with open(os.path.join(labels, 'images.txt'), 'w') as f:
        f.write(''.join(f'{i + 1} {p}\n' for i, p in enumerate(names)))
    with open(os.path.join(labels, 'image_class_labels.txt'), 'w') as f:
        f.write(''.join(f'{i + 1} {i % 200 + 1}\n' for i in range(n)))
    os.makedirs(os.path.join(root, 'mesh_templates'))
    write_uvsphere_obj(os.path.join(root, 'mesh_templates', 'uvsphere_16rings.obj'), rings=16)


def driver_epochs(argv, epochs):
    """Epoch times from the 'Time per epoch' lines of one main.main run."""
    import main
    main.main(argv + ['--epochs', str(epochs)])
    with open(os.path.join('gan_weights', argv[1], 'log.txt')) as f:
        return [float(line.split()[3]) for line in f if line.startswith('Time per epoch')]


def direct_epochs(argv, epochs):
    import main
    from gan_training import GANTrainer
    from rendering.mesh_template import MeshTemplate
    args = main.build_parser().parse_args(argv + ['--epochs', str(epochs)])
    ds = main.make_dataset(args)
    main.derive_settings(args, ds)
    ds.to_device('cuda')
    gan = GANTrainer(args, mesh_template=MeshTemplate(args.mesh_path, is_symmetric=args.symmetric_g, device='cuda'))
    times = []
    while gan.epoch < args.epochs:
        start = time.time()
        gan.train_epoch(ds.train_batches(args.batch_size, gan.epoch, seed=0))
        times.append(time.time() - start)
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=100)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--epochs', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_drivers: needs a CUDA device')
    B = 32
    root = tempfile.mkdtemp()
    write_tree(root, a.iters * B)
    os.chdir(root)
    argv = ['--weights', 't', '--dataset', 'cub', '--texture_resolution', '256', '--batch_size', str(B),
            '--save_freq', '1000', '--checkpoint_freq', '1000', '--evaluate_freq', '1000']
    rates = {'driver': [], 'direct': []}
    for _ in range(a.rounds):
        for name, fn in (('driver', driver_epochs), ('direct', direct_epochs)):
            t = fn(argv, a.epochs)[1:]
            rates[name] += [a.iters / x for x in t]
            torch.cuda.empty_cache()
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip()
    print(json.dumps(dict(gpu=q, iters_per_epoch=a.iters, batch=B,
                          driver_it_s=rates['driver'], direct_it_s=rates['direct'],
                          driver_median=float(np.median(rates['driver'])), direct_median=float(np.median(rates['direct'])))))


if __name__ == '__main__':
    main()
