"""GAN training data: the pseudo-ground-truth datasets main.py trains and evaluates on (reference: data/abstract_dataset.py),
and their device path.

Host side, same behaviour as the reference: `__getitem__` loads one record (`data.pseudo_gt.load_pseudo_ground_truth`),
drops the image and mirrors the maps in UV space with probability 1/2 (`mirror_tex`) unless augmentation is off or
args.evaluate; `AbstractDatasetForEvaluation` returns poses, class, and the whole record.  A plain DataLoader over these
works as in the reference.

Device path: `to_device()` packs every record once into fp16 / fp32 planes (device memory, or pinned host memory read over
PCIe); a training or evaluation batch is then ONE `b3d_gather_fields` launch (gather, fp16 -> fp32, mirror) with no host
work, no host-to-device copy and no synchronisation per batch.
    ds.to_device()
    gan.train_epoch(ds.train_batches(args.batch_size, gan.epoch))
    evaluator.evaluate(ds.eval_batches(args.batch_size))
Two deliberate differences from a DataLoader over the host dataset: the flips are one seeded Bernoulli(1/2) draw per sample
per epoch (the reference draws each flip from the loader worker's global RNG, so its stream depends on num_workers; the
distribution is the same), and the shuffle is seeded explicitly from (seed, epoch) instead of the global RNG.
"""
import glob
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from torch.utils.data import DistributedSampler, RandomSampler

from data.pseudo_gt import load_poses_metadata, load_pseudo_ground_truth, mirror_tex, pseudo_gt_dir

_FLIP_STREAM = 0x5EED_F11B


def epoch_seed(seed, epoch, rank=0):
    """The torch generator seed of one (seed, epoch, rank)."""
    return (int(seed) * 1_000_003 + int(epoch)) * 1_009 + int(rank) & ((1 << 63) - 1)


def epoch_order(n, epoch, seed=0, rank=0, world=1):
    """The sample order of one epoch, as main.py's shuffled loader draws it: single process, torch's RandomSampler with a
    generator seeded from (seed, epoch); under torch.distributed, DistributedSampler(shuffle=True, seed=seed) after
    set_epoch(epoch) (the rank's share, padded to equal length across ranks as the sampler does).  -> int64 [len]."""
    if world == 1:
        g = torch.Generator()
        g.manual_seed(epoch_seed(seed, epoch))
        return torch.tensor(list(RandomSampler(range(n), generator=g)), dtype=torch.int64)
    s = DistributedSampler(range(n), num_replicas=world, rank=rank, shuffle=True, seed=seed)
    s.set_epoch(epoch)
    return torch.tensor(list(s), dtype=torch.int64)


def epoch_flips(count, epoch, seed=0, rank=0):
    """One Bernoulli(1/2) mirror decision per position of the epoch's order.  -> uint8 [count]."""
    g = torch.Generator()
    g.manual_seed(epoch_seed(seed, epoch, rank) ^ _FLIP_STREAM)
    return torch.randint(0, 2, (count,), generator=g, dtype=torch.uint8)


def eval_shard(n, rank=0, world=1):
    """Contiguous [start, end) share of rank: every index exactly once across ranks, no padding."""
    return rank * n // world, (rank + 1) * n // world


def _raw_record(directory, idx):
    return np.load(os.path.join(directory, f'{idx}.npz'), allow_pickle=True)['data'].item()


class AbstractDataset(torch.utils.data.Dataset):
    def __init__(self, args, augment=True, root=''):
        """args: dataset, texture_resolution, evaluate, conditional_class (and conditional_color for P3D).
        root: directory holding cache/<dataset> and datasets/ (default: the working directory, as in the reference)."""
        if getattr(args, 'conditional_text', False):
            raise ValueError('conditional_text is not supported: the text-conditioned path of the reference is not '
                             'functional (it needs a caption encoder that its datasets never set up)')
        self.args, self.root, self.augment = args, root, augment
        self.cache_dir = os.path.join(root, 'cache', args.dataset)
        self.data = load_poses_metadata(self.cache_dir)
        n = len(self.data['path'])
        found = len(glob.glob(os.path.join(pseudo_gt_dir(self.cache_dir, args.texture_resolution), '*.npz')))
        if found not in (0, n):
            raise ValueError(f'{pseudo_gt_dir(self.cache_dir, args.texture_resolution)} holds {found} pseudo-ground-truth '
                             f'files for {n} poses; re-export it')
        self.has_pseudo_ground_truth = found == n
        if not self.has_pseudo_ground_truth and not args.evaluate:
            raise ValueError('training needs the pseudo-ground-truth: export it first (InverseRenderer + '
                             'data.pseudo_gt.save_pseudo_gt)')
        self.store = None

    def name(self):
        raise NotImplementedError()

    def suggest_truncation_sigma(self):
        raise NotImplementedError()

    def suggest_num_discriminators(self):
        raise NotImplementedError()

    def suggest_mesh_template(self):
        raise NotImplementedError()

    def __len__(self):
        return len(self.data['path'])

    def record_index(self, idx):
        """File index of sample idx in the pseudo-ground-truth directory."""
        return idx

    def load_pseudo_ground_truth(self, idx):
        return load_pseudo_ground_truth(self.cache_dir, self.args.texture_resolution, self.record_index(idx))

    def __getitem__(self, idx):
        d = self.load_pseudo_ground_truth(idx)
        del d['image']
        if self.augment and not self.args.evaluate and torch.randint(0, 2, size=(1,)).item() == 1:
            d = {k: mirror_tex(v) for k, v in d.items()}
        if self.args.conditional_class:
            d['class'] = self.classes[idx]
        d['idx'] = idx
        return d

    mirror_tex = staticmethod(mirror_tex)

    # ------------------------------------------------------------------------------------------------ device store
    def _pgt_dir(self):
        return pseudo_gt_dir(self.cache_dir, self.args.texture_resolution)

    def store_layout(self, include_image=False):
        """{field: (shape, dtype)} of the packed store: the record planes (dtype as stored: fp16 textures, fp32 mesh map),
        the first three image channels with include_image, and the int64 class rows when conditional."""
        n = len(self)
        lay = {}
        if self.has_pseudo_ground_truth:
            rec = _raw_record(self._pgt_dir(), self.record_index(0))
            for k in ('texture', 'texture_alpha', 'mesh'):
                lay[k] = ((n,) + tuple(rec[k].shape), rec[k].dtype)
            if include_image:
                lay['image'] = ((n, 3) + tuple(rec['image'].shape[1:]), rec['image'].dtype)
        elif include_image:
            raise ValueError('include_image needs the pseudo-ground-truth records')
        if self.args.conditional_class:
            lay['class'] = ((n, len(self.classes[0])), torch.int64)
        return lay

    def packed_bytes(self, include_image=False):
        """Bytes of the packed store (the poses and index buffers, 36 bytes per sample, not counted)."""
        return sum(int(np.prod(s)) * torch.empty(0, dtype=d).element_size() for s, d in self.store_layout(include_image).values())

    def to_device(self, device='cuda', storage='device', include_image=False, workers=8, chunk=64):
        """Pack every record into one store per field.  storage='device': device memory (checked against the free memory
        first); 'host': pinned host memory that the gather kernel reads over PCIe, for stores that do not fit beside
        training.  Records are read `chunk` at a time by `workers` threads, so the host holds one chunk besides the store.
        Under torch.distributed every rank packs its own full copy (the sampler reshuffles across ranks every epoch).
        -> self."""
        import b3d
        if storage not in ('device', 'host'):
            raise ValueError(f"storage={storage!r}: expected 'device' or 'host'")
        device = torch.device(device)
        if device.type != 'cuda' or not torch.cuda.is_available():
            raise b3d.B3DError(f'to_device({device}): the packed store is read by a CUDA kernel and needs a CUDA device; '
                               'there is no CPU fallback')
        lay = self.store_layout(include_image)
        need = self.packed_bytes(include_image)
        if storage == 'device':
            free, _ = torch.cuda.mem_get_info(device)
            if need > free:
                raise b3d.B3DError(f'to_device: the packed store needs {need} bytes, {free} are free on {device}; '
                                   "storage='host' keeps it in pinned host memory instead")
        planes = [k for k in ('texture', 'texture_alpha', 'mesh', 'image') if k in lay]
        store = {k: (torch.empty(s, dtype=d, device=device) if storage == 'device' else torch.empty(s, dtype=d, pin_memory=True))
                 for k, (s, d) in lay.items() if k in planes}
        n, directory = len(self), self._pgt_dir()

        def load(i):
            rec = _raw_record(directory, self.record_index(i))
            return [rec[k][:3] if k == 'image' else rec[k] for k in planes]

        with ThreadPoolExecutor(max_workers=workers) as pool:
            for a in range(0, n, chunk):
                recs = list(pool.map(load, range(a, min(a + chunk, n))))
                for j, k in enumerate(planes):
                    store[k][a:a + len(recs)].copy_(torch.stack([r[j] for r in recs]))
        if 'class' in lay:
            store['class'] = torch.as_tensor(np.stack(self.classes), dtype=torch.int64).to(device)
        for k in ('scale', 'translation', 'rotation'):
            store[k] = torch.as_tensor(self.data[k]).to(device=device, dtype=torch.float32).contiguous()
        store['arange'] = torch.arange(n, dtype=torch.int32, device=device)
        self.store, self.store_device, self.storage = store, device, storage
        torch.cuda.synchronize(device)
        return self

    def _require_store(self):
        if self.store is None:
            raise RuntimeError('call to_device() first')
        return self.store

    def batch_outputs(self, batch_size):
        """Fresh output tensors of one training batch: the keyword arguments of GANTrainer.step."""
        st, dev = self._require_store(), self.store_device
        out = {'X_tex': torch.empty((batch_size,) + st['texture'].shape[1:], device=dev),
               'X_alpha': torch.empty((batch_size,) + st['texture_alpha'].shape[1:], device=dev),
               'X_mesh': None if getattr(self.args, 'texture_only', False) else torch.empty((batch_size,) + st['mesh'].shape[1:], device=dev),
               'C': None}
        if self.args.conditional_class:
            out['C'] = torch.empty((batch_size,) + st['class'].shape[1:], dtype=torch.int64, device=dev)
        return out

    def _gather_train(self, idx, flip, out):
        from b3d.data import gather_fields
        st = self.store
        fields = [(st['texture'], out['X_tex'], True, 1.0, 0.0), (st['texture_alpha'], out['X_alpha'], True, 1.0, 0.0)]
        if out.get('X_mesh') is not None:
            fields.append((st['mesh'], out['X_mesh'], True, 1.0, 0.0))
        if out.get('C') is not None:
            fields.append((st['class'], out['C'], False, 1.0, 0.0))
        gather_fields(fields, idx, flip)
        return out

    def gather(self, idx, flip=None, out=None):
        """One training batch of the samples idx (int32 CUDA [B]) mirrored where flip (uint8 CUDA [B] or None) is set,
        written into `out` (static tensors from batch_outputs() for CUDA-graph capture: copy the step's indices into a
        static idx / flip device-to-device before replay) or into fresh tensors.  Outside a capture the indices are
        range-checked first (one synchronisation); inside one, an out-of-range index yields NaN rows (class -1)."""
        import b3d
        st = self._require_store()
        if not self.has_pseudo_ground_truth:
            raise ValueError('training batches need the pseudo-ground-truth records')
        if not torch.cuda.is_current_stream_capturing() and idx.numel():
            lo, hi = int(idx.min()), int(idx.max())
            if lo < 0 or hi >= len(self):
                raise b3d.B3DError(f'gather: index range [{lo}, {hi}] outside the {len(self)} samples')
        return self._gather_train(idx, flip, out if out is not None else self.batch_outputs(idx.shape[0]))

    def train_batches(self, batch_size, epoch, seed=0, rank=0, world=1):
        """The epoch's training batches, as GANTrainer.step's keyword dicts (X_tex, X_alpha, X_mesh (None with
        texture_only), C (None unless conditional_class)): order from epoch_order, batches of batch_size with the last
        partial one dropped (main.py's drop_last=True), flips from epoch_flips unless augmentation is off or
        args.evaluate.  The order and flips are uploaded once; each batch is one gather launch."""
        self._require_store()
        if not self.has_pseudo_ground_truth:
            raise ValueError('training batches need the pseudo-ground-truth records')
        order = epoch_order(len(self), epoch, seed, rank, world)
        dev = self.store_device
        idx = order.to(torch.int32).to(dev)
        flips = epoch_flips(len(order), epoch, seed, rank).to(dev) if self.augment and not self.args.evaluate else None
        for k in range(len(order) // batch_size):
            s = slice(k * batch_size, (k + 1) * batch_size)
            yield self._gather_train(idx[s], flips[s] if flips is not None else None, self.batch_outputs(batch_size))

    def eval_batches(self, batch_size, rank=0, world=1):
        """The evaluation loader's batches (AbstractDatasetForEvaluation collated, sequential, never mirrored, last batch
        ragged) over rank's contiguous shard: idx, rotation, scale, translation, class (conditional), and with
        pseudo-ground-truth texture, texture_alpha, mesh, plus image (RGB in [0, 1]) when packed.  All on the device."""
        from b3d.data import gather_fields
        st = self._require_store()
        dev = self.store_device
        start, end = eval_shard(len(self), rank, world)
        for a in range(start, end, batch_size):
            b = min(a + batch_size, end)
            d = {'scale': st['scale'][a:b], 'translation': st['translation'][a:b], 'rotation': st['rotation'][a:b],
                 'idx': torch.arange(a, b, dtype=torch.int64, device=dev)}
            if 'class' in st:
                d['class'] = st['class'][a:b]
            fields = []
            for k in ('image', 'texture', 'texture_alpha', 'mesh'):
                if k in st:
                    shape = (b - a, 3 if k == 'image' else st[k].shape[1]) + tuple(st[k].shape[2:])
                    d[k] = torch.empty(shape, device=dev)
                    fields.append((st[k], d[k], False, 0.5 if k == 'image' else 1.0, 0.5 if k == 'image' else 0.0))
            if fields:
                gather_fields(fields, st['arange'][a:b])
            yield d


class AbstractDatasetForEvaluation(torch.utils.data.Dataset):
    def __init__(self, dataset):
        self.dataset = dataset

    def __len__(self):
        return len(self.dataset)

    def __getitem__(self, idx):
        ds = self.dataset
        d = {'scale': ds.data['scale'][idx], 'translation': ds.data['translation'][idx],
             'rotation': ds.data['rotation'][idx], 'idx': idx}
        if ds.args.conditional_class:
            d['class'] = ds.classes[idx]
        if ds.has_pseudo_ground_truth:
            d.update(ds.load_pseudo_ground_truth(idx))
        return d
