"""The synthetic pseudo-ground-truth caches behind tests/golden/dataset_reference.npz, shared by the generator and the tests:
`make_inputs` draws them (seeded), `write_tree` lays them out on disk in the reference's format under a root directory:
    cache/<cub|p3d>/poses_metadata.npz, cache/<cub|p3d>/pseudogt_<R>x<R>/<idx>.npz,
    datasets/cub/CUB_200_2011/images.txt + image_class_labels.txt, datasets/p3d/p3d_labels.csv."""
import os
from types import SimpleNamespace

import numpy as np
import torch

R = 32           # pseudo-GT resolution
N = 12           # poses per dataset
IMG = 24         # stored image size


def make_inputs(seed=0, res=R, n=N, img=IMG):
    """Records of n poses per dataset at pseudo-GT resolution res (the golden: res=R, n=N=12)."""
    assert n <= 12
    g = torch.Generator().manual_seed(seed)
    out = {}
    for ds, img_c in (('cub', 4), ('p3d', 3)):
        # values on coarse grids (exact in fp16, so the fixture compresses well); textures masked like the exporter's
        # (negative texels times a zero mask give -0.0)
        mask = (torch.rand(n, 1, res, res, generator=g) > 0.3).float()
        out[f'{ds}_texture'] = (torch.randint(-4, 5, (n, 3, res, res), generator=g) / 4 * mask).half().numpy()
        out[f'{ds}_texture_alpha'] = (torch.randint(0, 5, (n, 1, res, res), generator=g) / 4 * mask).half().numpy()
        out[f'{ds}_mesh'] = (torch.randint(-4, 5, (n, 3, 32, 32), generator=g) / 64).numpy()
        out[f'{ds}_image'] = (torch.randint(-4, 5, (n, img_c, img, img), generator=g) / 4).half().numpy()
        out[f'{ds}_scale'] = (0.5 + torch.rand(n, 1, generator=g)).numpy()
        out[f'{ds}_translation'] = (torch.randn(n, 3, generator=g) * 0.1).numpy()
        out[f'{ds}_rotation'] = torch.nn.functional.normalize(torch.randn(n, 4, generator=g), dim=1).numpy()
    # CUB: 15 images in images.txt, 12 of them posed, labels 1-based over a few species
    cub_names = [f'{(i % 5) + 1:03d}.Species_{(i % 5) + 1}/Bird_{i:04d}.jpg' for i in range(15)]
    posed = [cub_names[i] for i in (3, 0, 7, 14, 1, 9, 11, 2, 5, 13, 6, 10)][:n]
    out['cub_path'] = np.array(posed)
    out['cub_images_txt'] = np.array(''.join(f'{i + 1} {p}\n' for i, p in enumerate(cub_names)))
    out['cub_labels_txt'] = np.array(''.join(f'{i + 1} {(i * 7) % 200 + 1}\n' for i in range(15)))
    # P3D: ImageNet and PASCAL paths interleaved; the csv lists every file (header, then filename,col1,col2,shape,extra)
    paths = [f'car_imagenet/n02814533_{i:05d}.JPEG' if i % 3 != 1 else f'car_pascal/2008_{i:06d}.jpg' for i in range(n)]
    out['p3d_path'] = np.array(paths)
    cols, shapes = ['red', 'blue', 'white', 'black'], ['sedan', 'suv', 'hatchback']
    rows = [f'{p.split("/")[-1]},{cols[i % 4]},{cols[(i * 3 + 1) % 4]},{shapes[(i * 5) % 3]},x' for i, p in enumerate(paths)]
    out['p3d_csv'] = np.array('filename,color1,color2,shape,extra\n' + '\n'.join(rows) + '\n')
    return out


def write_tree(root, inp, datasets=('cub', 'p3d'), with_pseudo_gt=True, drop_file=None):
    """Write the caches under root.  drop_file=(dataset, idx) leaves one record out (count mismatch)."""
    for ds in datasets:
        cache = os.path.join(root, 'cache', ds)
        os.makedirs(cache, exist_ok=True)
        np.savez_compressed(os.path.join(cache, 'poses_metadata'), data={
            'scale': torch.from_numpy(inp[f'{ds}_scale']), 'translation': torch.from_numpy(inp[f'{ds}_translation']),
            'rotation': torch.from_numpy(inp[f'{ds}_rotation']), 'path': [str(p) for p in inp[f'{ds}_path']]})
        if with_pseudo_gt:
            res = inp[f'{ds}_texture'].shape[-1]
            d = os.path.join(cache, f'pseudogt_{res}x{res}')
            os.makedirs(d, exist_ok=True)
            for i in range(len(inp[f'{ds}_path'])):
                if drop_file == (ds, i):
                    continue
                np.savez_compressed(os.path.join(d, f'{i}'), data={
                    k: torch.from_numpy(inp[f'{ds}_{k}'][i].copy()) for k in ('mesh', 'texture', 'texture_alpha', 'image')})
    cub = os.path.join(root, 'datasets', 'cub', 'CUB_200_2011')
    os.makedirs(cub, exist_ok=True)
    with open(os.path.join(cub, 'images.txt'), 'w') as f:
        f.write(str(inp['cub_images_txt']))
    with open(os.path.join(cub, 'image_class_labels.txt'), 'w') as f:
        f.write(str(inp['cub_labels_txt']))
    os.makedirs(os.path.join(root, 'datasets', 'p3d'), exist_ok=True)
    with open(os.path.join(root, 'datasets', 'p3d', 'p3d_labels.csv'), 'w') as f:
        f.write(str(inp['p3d_csv']))


def make_args(ds, **kw):
    a = dict(dataset=ds, texture_resolution=R, evaluate=False, conditional_class=True, conditional_text=False,
             conditional_color=ds == 'p3d', texture_only=False)
    a.update(kw)
    return SimpleNamespace(**a)
