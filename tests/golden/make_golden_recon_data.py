"""Generate tests/golden/recon_data_reference.npz by RUNNING the reference's CMR loaders (authoring container only):
    python tests/golden/make_golden_recon_data.py
It reads no other golden and runs on its own, beside regenerate_all.sh (which does not list it).
The reference's cmr_data.cub.CUBDataset and cmr_data.p3d.P3dDataset are imported unmodified from the reference tree, and
run_reconstruction.py's ImageDataset is executed from the script's syntax tree.  skimage is absent here: a stand-in module
supplies skimage.io.imread through PIL (what skimage's imread does for these files).  The modules' __file__ is pointed into a
temporary tree so their '../datasets/...' paths resolve to the synthetic annotations and PNG photos of
recon_data_common.write_tree.  OpenCV (cv2.resize) is the installed 4.13.

Recorded per dataset, with the module's torch.randint patched to force the mirror draw (0, then 1), at img_size R = 32 for
every item and at the list [32, 37, 64] for every item: the items' sfm_pose, kp, mirrored, inds, path, and the images as
fp32 (item 'img' and 'mask' rounded once).  Stored once each: the mirrored images are the unmirrored ones column-reversed, the
list form's first resolution equals the single form, and ImageDataset's tuple is (fp32(img) * 2 - 1) * fp32(mask), mask,
the pose and the index: all checked bit for bit here.  Nothing of the reference is copied into the repository."""
import ast
import os
import sys
import tempfile
import types

import numpy as np
import torch
from PIL import Image

REF = "/root/reference/code"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import recon_data_common as RD                                # noqa: E402


def imread(path):
    with Image.open(path) as im:
        return np.asarray(im)                                   # 'L' -> [H, W], 'RGB' -> [H, W, 3], as skimage


skimage = types.ModuleType('skimage')
skimage.io = types.ModuleType('skimage.io')
skimage.io.imread = imread
sys.modules['skimage'], sys.modules['skimage.io'] = skimage, skimage.io
sys.path.insert(0, REF)
import cmr_data.base as ref_base                              # noqa: E402  (reference)
import cmr_data.cub as ref_cub                                # noqa: E402  (reference)
import cmr_data.p3d as ref_p3d                                # noqa: E402  (reference)


def image_dataset_class():
    tree = ast.parse(open(os.path.join(REF, 'run_reconstruction.py')).read())
    node = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == 'ImageDataset')
    ns = {'torch': torch, 'np': np}
    exec(compile(ast.Module(body=[node], type_ignores=[]), 'run_reconstruction.py', 'exec'), ns)
    return ns['ImageDataset']


ImageDataset = image_dataset_class()
_randint = torch.randint


def forced(f):
    return lambda *a, **k: torch.tensor([f])


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint64)


def make(ds_name, tmp, img_size):
    mod = ref_cub if ds_name == 'cub' else ref_p3d
    mod.__file__ = os.path.join(tmp, 'cmr_data', os.path.basename(mod.__file__))
    if ds_name == 'cub':
        return ref_cub.CUBDataset('train', True, img_size)
    return ref_p3d.P3dDataset('train', True, img_size)


def record(ds_name, tmp, out):
    single, multi = {}, {}
    for f in (0, 1):
        for img_size, dst in ((RD.R, single), (list(RD.SIZES), multi)):
            ds = make(ds_name, tmp, img_size)
            wrap = ImageDataset(ds, img_size)
            torch.randint = forced(f)
            try:
                items = [ds[i] for i in range(len(ds))]
                tuples = [wrap[i] for i in range(len(ds))]
            finally:
                torch.randint = _randint
            dst[f] = (items, tuples, wrap.paths)
    n = len(single[0][0])
    for f in (0, 1):
        items, tuples, paths = single[f]
        assert [it['mirrored'] for it in items] == [bool(f)] * n and [it['inds'] for it in items] == list(range(n))
        out[f'{ds_name}_flip{f}_sfm_pose'] = np.stack([it['sfm_pose'] for it in items])
        out[f'{ds_name}_flip{f}_kp'] = np.stack([it['kp'] for it in items])
        img = np.stack([it['img'] for it in items]).astype(np.float32)
        mask = np.stack([it['mask'] for it in items]).astype(np.float32)
        if f == 0:
            out[f'{ds_name}_img'], out[f'{ds_name}_mask'] = img, mask
            out[f'{ds_name}_paths'] = np.array(paths)
            assert [it['path'] for it in items] == paths
        else:
            assert np.array_equal(bits(img), bits(out[f'{ds_name}_img'][..., ::-1]))
            assert np.array_equal(bits(mask), bits(out[f'{ds_name}_mask'][..., ::-1]))
        for i, t in enumerate(tuples):
            X, scale, trans, rot, ind = (v.numpy() for v in t)
            want = (img[i] * 2 - 1) * mask[i][None]
            assert np.array_equal(bits(X[:3]), bits(want)) and np.array_equal(bits(X[3]), bits(mask[i]))
            pose = items[i]['sfm_pose']
            assert np.array_equal(bits(scale), bits(pose[:1].astype(np.float32)))
            assert np.array_equal(bits(trans), bits(np.array([pose[1], pose[2], 0], np.float32)))
            assert np.array_equal(bits(rot), bits(pose[3:].astype(np.float32)))
            assert ind.tolist() == [i + n * f]
        # the list form: the same first resolution and pose, one masked image per extra size
        m_items, m_tuples, _ = multi[f]
        for i in range(n):
            assert np.array_equal(bits(m_items[i]['sfm_pose']), bits(items[i]['sfm_pose']))
            assert np.array_equal(bits(m_items[i]['img'].astype(np.float32)), bits(img[i]))
            for k, t in zip(RD.SIZES[1:], m_tuples[i][1:len(RD.SIZES)]):
                img_k, mask_k = m_items[i][f'img_{k}']
                img_k, mask_k = img_k.astype(np.float32), mask_k.astype(np.float32)
                if f == 0:
                    out.setdefault(f'{ds_name}_img_{k}', []).append(img_k)
                    out.setdefault(f'{ds_name}_mask_{k}', []).append(mask_k)
                else:
                    assert np.array_equal(bits(img_k), bits(out[f'{ds_name}_img_{k}'][i][..., ::-1]))
                assert np.array_equal(bits(t.numpy()), bits((img_k * 2 - 1) * mask_k[None]))
            assert len(m_tuples[i]) == 4 + len(RD.SIZES)
        if f == 0:
            for k in RD.SIZES[1:]:
                out[f'{ds_name}_img_{k}'] = np.stack(out[f'{ds_name}_img_{k}'])
                out[f'{ds_name}_mask_{k}'] = np.stack(out[f'{ds_name}_mask_{k}'])
    # the validation form is never mirrored
    ds = make(ds_name, tmp, RD.R)
    ds.is_train = False
    out[f'{ds_name}_val_mirrored'] = np.array([ds[i]['mirrored'] for i in range(n)])


def main():
    inp = RD.make_inputs()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        RD.write_tree(tmp, inp)
        os.makedirs(os.path.join(tmp, 'cmr_data'))
        for ds_name in RD.LAYOUT:
            record(ds_name, tmp, out)
    path = os.path.join(HERE, 'recon_data_reference.npz')
    np.savez_compressed(path, **{f'in_{k}': v for k, v in inp.items()}, **out)
    print(f'wrote {path} ({os.path.getsize(path)} bytes)')


if __name__ == '__main__':
    main()
