"""The synthetic CUB / PASCAL3D+ trees behind tests/golden/recon_data_reference.npz, shared by the generator and the tests:
`make_inputs` draws them (seeded), `write_tree` lays them out under a root directory in the layout of the shipped
annotations (scipy.io.savemat structs) with lossless PNG photos:
    datasets/cub/data/<split>_cub_cleaned.mat, datasets/cub/sfm/anno_<split>.mat, datasets/cub/CUB_200_2011/images/...
    datasets/p3d/data/car_<split>.mat, car_kps.mat, datasets/p3d/sfm/car_<split>.mat, datasets/p3d/PASCAL3D+_release1.1/Images/...
The boxes are chosen to cover: every photo border crossed (background fill), a box larger than its photo, tall and wide
boxes, padded edges at .5 (Python's round to even in square_bbox) and odd side differences (.5 centring), crop sides that
are upscaled (S < R), halved exactly (S = 2R) and downscaled by a non-integer factor (83 -> 37); one grey photo per dataset;
rotations with w the largest quaternion component and with x, y, z the largest (both branches of the conversion)."""
import os

import numpy as np
import scipy.io as sio
from PIL import Image

R = 32                       # img_size of the single-resolution items
SIZES = [32, 37, 64]         # the list form (--generate_pseudogt's [256, 299, 1024], scaled down)
SPLIT = {'cub': 'train', 'p3d': 'train'}
NKP = {'cub': 15, 'p3d': 12}
P3D_KP_PERM = np.array([5, 6, 7, 8, 1, 2, 3, 4, 11, 12, 9, 10], np.uint8)    # 1-based, as car_kps.mat

# (photo h, w, grey, box x1, y1, x2, y2 (1-based, inclusive), rotation axis, angle in degrees)
LAYOUT = {
    'cub': [
        (60, 80, False, -3, 12, 54, 40, 'z', 30),      # crosses the left border; wide; S = 64 (exact 2x down to 32)
        (80, 56, False, 10, -6, 40, 68, 'x', 170),     # crosses the top border; tall; S = 83 (83 -> 37, 83 -> 64)
        (48, 64, False, 50, 20, 67, 34, 'y', 175),     # crosses the right border; S = 20 (upscaled to 32, 37, 64)
        (50, 60, True, 20, 30, 49, 55, 'z', 179),      # grey photo; crosses the bottom border
        (40, 50, False, 11, 11, 20, 24, 'xy', 60),     # width 10: padded edges at .5; odd side difference
        (30, 36, False, -5, -4, 45, 40, 'xyz', 120),   # box larger than the photo: every border
        (64, 64, False, 8, 17, 37, 44, 'yz', -100),    # width 30: pad 1.5, .5 rounding on both edges
    ],
    'p3d': [
        (56, 72, False, 5, 10, 70, 48, 'z', -45),      # wide, near the right border; S = 72
        (70, 50, True, 12, -2, 41, 69, 'x', 178),      # grey; tall; crosses the top border
        (44, 60, False, -8, 3, 30, 38, 'y', 91),       # crosses the left border
        (60, 60, False, 40, 42, 66, 70, 'xz', 150),    # crosses the right and bottom borders
        (36, 40, False, 15, 14, 24, 27, 'xyz', -170),  # width 10: .5 padding; upscaled
    ],
}
CUB_KP_VIS = 11             # keypoints visible per item (the others are (0, 0, 0))


def rotation(axis, deg):
    """3x3 rotation by deg about the normalised axis ('x', 'xy', ...), float64."""
    v = np.array([c in axis for c in 'xyz'], float)
    v /= np.linalg.norm(v)
    t = np.deg2rad(deg)
    K = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])
    return np.eye(3) + np.sin(t) * K + (1 - np.cos(t)) * K @ K


def make_inputs(seed=0):
    g = np.random.default_rng(seed)
    out = {}
    for ds, layout in LAYOUT.items():
        n = len(layout)
        out[f'{ds}_n'] = np.array(n)
        for i, (h, w, grey, x1, y1, x2, y2, axis, deg) in enumerate(layout):
            yy, xx = np.mgrid[0:h, 0:w]
            base = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 255 // max(h - 1, 1)), ((xx + yy) * 7) % 256], -1)
            photo = np.clip(base + g.integers(-40, 41, (h, w, 3)), 0, 255).astype(np.uint8)
            out[f'{ds}_photo{i}'] = photo[..., 0] if grey else photo
            cy, cx = (y1 + y2) / 2 - 1, (x1 + x2) / 2 - 1
            ry, rx = max((y2 - y1) / 2, 1), max((x2 - x1) / 2, 1)
            blob = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1 + 0.3 * g.random((h, w))
            out[f'{ds}_mask{i}'] = blob.astype(np.uint8)
            out[f'{ds}_bbox{i}'] = np.array([x1, y1, x2, y2])
            nkp = NKP[ds]
            kp = np.zeros((3, nkp))
            vis = g.permutation(nkp) < (CUB_KP_VIS if ds == 'cub' else 8)
            kp[0, vis] = g.integers(1, w + 1, vis.sum())
            kp[1, vis] = g.integers(1, h + 1, vis.sum())
            kp[2, vis] = 1
            out[f'{ds}_parts{i}'] = kp.astype(np.uint16) if ds == 'cub' else kp
            out[f'{ds}_rot{i}'] = rotation(axis, deg)
            out[f'{ds}_scale{i}'] = np.array(20 + 60 * g.random())
            out[f'{ds}_trans{i}'] = np.array([x1 + (x2 - x1) * g.random(), y1 + (y2 - y1) * g.random()])
    return out


def rel_path(ds, i, grey=False):
    if ds == 'cub':
        return f'{(i % 3) + 1:03d}.Species_{(i % 3) + 1}/Bird_{i:04d}.png'
    return f'car_{"pascal" if i % 2 else "imagenet"}\\2008_{i:06d}.png'      # backslash as in the shipped files


def write_tree(root, inp):
    """The annotation files and photos of both datasets under root/datasets."""
    for ds in LAYOUT:
        n = int(inp[f'{ds}_n'])
        images = np.empty((1, n), dtype=[('rel_path', 'O'), ('bbox', 'O'), ('width', 'O'), ('height', 'O'),
                                         ('parts', 'O'), ('mask', 'O')])
        sfm = np.empty((1, n), dtype=[('rot', 'O'), ('scale', 'O'), ('trans', 'O')])
        top = os.path.join(root, 'datasets', ds)
        img_dir = os.path.join(top, 'CUB_200_2011', 'images') if ds == 'cub' else \
            os.path.join(top, 'PASCAL3D+_release1.1', 'Images')
        for i in range(n):
            photo, mask = inp[f'{ds}_photo{i}'], inp[f'{ds}_mask{i}']
            rp = rel_path(ds, i)
            path = os.path.join(img_dir, rp.replace('\\', '/'))
            os.makedirs(os.path.dirname(path), exist_ok=True)
            Image.fromarray(photo, 'L' if photo.ndim == 2 else 'RGB').save(path)
            x1, y1, x2, y2 = (int(v) for v in inp[f'{ds}_bbox{i}'])
            images[0, i] = (rp, {'x1': x1, 'y1': y1, 'x2': x2, 'y2': y2}, mask.shape[1], mask.shape[0],
                            inp[f'{ds}_parts{i}'], mask)
            sfm[0, i] = (inp[f'{ds}_rot{i}'], float(inp[f'{ds}_scale{i}']), inp[f'{ds}_trans{i}'])
        split = SPLIT[ds]
        os.makedirs(os.path.join(top, 'data'), exist_ok=True)
        os.makedirs(os.path.join(top, 'sfm'), exist_ok=True)
        if ds == 'cub':
            sio.savemat(os.path.join(top, 'data', f'{split}_cub_cleaned.mat'), {'images': images})
            sio.savemat(os.path.join(top, 'sfm', f'anno_{split}.mat'), {'sfm_anno': sfm})
        else:
            sio.savemat(os.path.join(top, 'data', f'car_{split}.mat'), {'images': images})
            sio.savemat(os.path.join(top, 'sfm', f'car_{split}.mat'), {'sfm_anno': sfm})
            sio.savemat(os.path.join(top, 'data', 'car_kps.mat'), {'kp_perm_inds': P3D_KP_PERM[:, None]})
