"""Generate tests/golden/dataset_reference.npz by RUNNING the reference's dataset classes (authoring container only):
    python tests/golden/make_golden_dataset.py
It reads no other golden and runs on its own, beside regenerate_all.sh (which does not list it).
The reference's data/abstract_dataset.py, cub_200_2011_dataset.py and pascal3d_plus_dataset.py are imported unmodified from
the reference tree and run with the working directory set to a temporary directory that holds a small synthetic cache in the
reference's on-disk format (dataset_common.write_tree: 12 poses per dataset, fp16 records at 32^2 with an 'image' field, CUB
label files, a P3D csv with ImageNet and PASCAL paths).  Recorded, for CUB and P3D (conditional class; P3D also colour):
every __getitem__ with the mirror branch taken and not taken (the module's torch.randint patched to return 1, then 0), every
AbstractDatasetForEvaluation item, one DataLoader batch over repeated indices with a fixed flip sequence, classes, n_classes,
the suggest_* values per conditioning / resolution, and the two ValueError cases (file count mismatch; no pseudo-GT while
training).  Stored: the synthetic inputs and these outputs, each once: the unmirrored items are the records widened to
fp32, the evaluation items' pseudo-GT planes are the unmirrored items, and the loader batch is the items of its (index, flip)
pairs (all three checked bit for bit here), so only the mirrored planes, the batch's indices, flips and classes, and the
evaluation poses, classes and images are stored beside the inputs.  Nothing of the reference is copied into the repository."""
import os
import sys
import tempfile

import numpy as np
import torch

REF = "/root/reference/code"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, REF)
import dataset_common as DC                                    # noqa: E402
from data.abstract_dataset import AbstractDatasetForEvaluation  # noqa: E402  (reference)
from data.cub_200_2011_dataset import CubDataset               # noqa: E402  (reference)
from data.pascal3d_plus_dataset import Pascal3DPlusDataset     # noqa: E402  (reference)

CLASSES = {'cub': CubDataset, 'p3d': Pascal3DPlusDataset}
BATCH_IDX = {'cub': [3, 0, 7, 7, 11, 2], 'p3d': [5, 0, 5, 7, 1]}
BATCH_FLIP = {'cub': [1, 0, 1, 0, 0, 1], 'p3d': [0, 1, 1, 0, 1]}

_randint = torch.randint


def fixed_randint(values):
    it = iter(values)
    return lambda *a, **k: torch.tensor([next(it)])


def stack(items, key, dtype=None):
    v = np.stack([np.asarray(it[key]) for it in items])
    return v.astype(dtype) if dtype else v


def as_fp16(a):
    """fp32 outputs whose values are exact in fp16 (the synthetic records use coarse grids) are stored as fp16, checked
    bit for bit (-0.0 included), to keep the fixture small."""
    h = a.astype(np.float16)
    assert np.array_equal(h.astype(np.float32).view(np.int32), a.view(np.int32))
    return h


def record(ds_name, inp, out):
    cls = CLASSES[ds_name]
    args = DC.make_args(ds_name)
    ds = cls(args)
    n = len(ds)
    out[f'{ds_name}_len'] = n
    out[f'{ds_name}_classes'] = np.stack(ds.classes)
    out[f'{ds_name}_n_classes'] = np.array(ds.n_classes)
    items = {}
    for f in (1, 0):
        torch.randint = fixed_randint([f] * n)
        items[f] = [ds[i] for i in range(n)]
        torch.randint = _randint
        assert [it['idx'] for it in items[f]] == list(range(n))
        out[f'{ds_name}_flip{f}_class'] = stack(items[f], 'class')
    # the mirrored items are stored; the unmirrored ones are the stored records widened to fp32 (checked here, and the
    # tests compare against the records)
    for k in ('texture', 'texture_alpha', 'mesh'):
        out[f'{ds_name}_flip1_{k}'] = as_fp16(stack(items[1], k))
        rec = inp[f'{ds_name}_{k}'][[ds.imagenet_indices[i] for i in range(n)] if ds_name == 'p3d' else slice(None)]
        assert np.array_equal(stack(items[0], k).view(np.int32), rec.astype(np.float32).view(np.int32)), k
    ev = AbstractDatasetForEvaluation(ds)
    evi = [ev[i] for i in range(n)]
    assert sorted(evi[0]) == sorted(['scale', 'translation', 'rotation', 'idx', 'class', 'image', 'texture',
                                       'texture_alpha', 'mesh'])
    for k in ('scale', 'translation', 'rotation', 'class'):
        out[f'{ds_name}_eval_{k}'] = stack(evi, k)
    out[f'{ds_name}_eval_image'] = as_fp16(stack(evi, 'image'))
    for k in ('texture', 'texture_alpha', 'mesh'):    # the unmirrored items
        assert np.array_equal(stack(evi, k).view(np.int32), stack(items[0], k).view(np.int32))
    # one collated batch of the reference's training loader over repeated indices
    idx = BATCH_IDX[ds_name]
    torch.randint = fixed_randint(BATCH_FLIP[ds_name])
    batch = next(iter(torch.utils.data.DataLoader(ds, batch_size=len(idx), sampler=idx)))
    torch.randint = _randint
    out[f'{ds_name}_batch_idx'] = np.array(idx)
    out[f'{ds_name}_batch_flip'] = np.array(BATCH_FLIP[ds_name])
    for k in ('texture', 'texture_alpha', 'mesh'):    # = the items of (index, flip), checked here
        want = np.stack([np.asarray((items[1] if f else items[0])[i][k]) for i, f in zip(idx, BATCH_FLIP[ds_name])])
        assert np.array_equal(batch[k].numpy().view(np.int32), want.view(np.int32)), k
    for k in ('class', 'idx'):
        out[f'{ds_name}_batch_{k}'] = batch[k].numpy()
    # suggest_* per conditioning and resolution
    sig = []
    for cc, col in ((False, False), (True, False), (True, True)):
        args.conditional_class, args.conditional_color = cc, col
        sig.append(ds.suggest_truncation_sigma())
    out[f'{ds_name}_sigma'] = np.array(sig)
    nd = []
    for r in (32, 256, 512, 1024):
        args.texture_resolution = r
        nd.append(ds.suggest_num_discriminators())
    out[f'{ds_name}_num_disc'] = np.array(nd)
    out[f'{ds_name}_template'] = np.array(ds.suggest_mesh_template())


def error_of(fn):
    try:
        fn()
    except Exception as e:                                     # noqa: BLE001
        return type(e).__name__
    return ''


def main():
    inp = DC.make_inputs()
    out = {}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        DC.write_tree(tmp, inp)
        os.chdir(tmp)
        try:
            for ds_name in CLASSES:
                record(ds_name, inp, out)
        finally:
            os.chdir(cwd)
    for ds_name, cls in CLASSES.items():
        with tempfile.TemporaryDirectory() as tmp:
            DC.write_tree(tmp, inp, datasets=(ds_name,), drop_file=(ds_name, 4))
            os.chdir(tmp)
            try:
                out[f'{ds_name}_err_count'] = np.array(error_of(lambda: cls(DC.make_args(ds_name))))
            finally:
                os.chdir(cwd)
        with tempfile.TemporaryDirectory() as tmp:
            DC.write_tree(tmp, inp, datasets=(ds_name,), with_pseudo_gt=False)
            os.chdir(tmp)
            try:
                out[f'{ds_name}_err_nopgt'] = np.array(error_of(lambda: cls(DC.make_args(ds_name))))
                ds = cls(DC.make_args(ds_name, evaluate=True))
                out[f'{ds_name}_nopgt_eval_len'] = len(ds)
                out[f'{ds_name}_nopgt_has'] = ds.has_pseudo_ground_truth
                out[f'{ds_name}_nopgt_eval_keys'] = np.array(sorted(AbstractDatasetForEvaluation(ds)[0]))
            finally:
                os.chdir(cwd)
    path = os.path.join(HERE, 'dataset_reference.npz')
    np.savez_compressed(path, **{f'in_{k}': v for k, v in inp.items()}, **out)
    print(f'wrote {path} ({os.path.getsize(path)} bytes)')


if __name__ == '__main__':
    main()
