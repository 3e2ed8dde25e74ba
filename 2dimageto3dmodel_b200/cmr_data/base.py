"""Image datasets of the reconstruction stage (reference: cmr_data/base.py): photo + annotation mask + SfM pose per item,
cropped to the padded square box, resized and optionally mirrored.

Host side, same behaviour as the reference: `__getitem__` decodes the photo, crops it and the mask to the box padded by 5 %
(pixels outside the photo: 1.0 in RGB, 0 in the mask), resizes both with OpenCV's float64 bilinear rule (restated in
numpy, `image_utils.resize`), mirrors with probability 1/2 on the training split (torch.randint per item), and returns
img, kp, mask, sfm_pose, mirrored, inds, path and img_<res> for every extra resolution.  A plain DataLoader over
`ImageDataset(ds, img_size)` works as in run_reconstruction.py.  Photos are decoded with PIL (convert('RGB')).

Device path: `to_device()` decodes every photo once and keeps only the crop window inside the photo, as RGBM bytes (one
32-bit word per pixel), in one device buffer, with a pose table [N, 2, 8] (unmirrored / mirrored: scale, tx, ty, 0, q)
computed here in float64 and rounded to fp32 once.  A batch is then ONE `b3d_image_batch` launch (crop, resize in double,
mirror, the ImageDataset arithmetic, poses and indices) with no host work, no host-to-device copy and no synchronisation
per batch:
    ds.to_device()
    recon.train_epoch(ds.train_batches(args.batch_size, recon.epoch))
    recon.evaluate(val_ds.eval_batches(args.batch_size))
Deliberate difference from the reference's loader: the flips and the shuffle are seeded per epoch (`epoch_flips`,
`epoch_order`) instead of drawn from the loader workers' global RNG.
"""
import copy
import os.path as osp
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from PIL import Image
from torch.utils.data import Dataset

from data.abstract_dataset import epoch_flips, epoch_order, eval_shard

from . import image_utils
from . import transformations

_MIRROR = np.diag([-1, 1, 1, 1])


def imread_rgb(path):
    """The photo as float64 RGB in [0, 1] (grey photos replicated to three channels, as the reference does)."""
    with Image.open(path) as im:
        return np.asarray(im.convert('RGB')) / 255.0


def imread_rgb_u8(path):
    with Image.open(path) as im:
        return np.asarray(im.convert('RGB'))


class BaseDataset(Dataset):
    """img, mask, kp, pose data loader.  Subclasses set kp_perm, img_dir, anno, anno_sfm and num_imgs."""

    def __init__(self, is_train, img_size):
        self.img_sizes = list(img_size) if isinstance(img_size, list) else [img_size]
        self.jitter_frac = 0
        self.padding_frac = 0.05
        self.is_train = is_train
        self.store = None

    def get_paths(self):
        return [str(data.rel_path).replace('\\', '/') for data in self.anno]

    def image_path(self, index):
        return osp.join(self.img_dir, str(self.anno[index].rel_path)).replace('\\', '/')

    # -------------------------------------------------------------------------------------------------- host items
    def crop_box(self, index):
        """The square crop box [x0, y0, x0 + S - 1, y0 + S - 1] of item index (zero-indexed, padded, squared)."""
        data = self.anno[index]
        bbox = np.array([data.bbox.x1, data.bbox.y1, data.bbox.x2, data.bbox.y2], float) - 1
        bbox = image_utils.peturb_bbox(bbox, pf=self.padding_frac, jf=self.jitter_frac if self.is_train else 0)
        return image_utils.square_bbox(bbox)

    def sfm_pose(self, index):
        """[scale, trans [2], quaternion [4]] of the SfM annotation, float64."""
        data_sfm = self.anno_sfm[index]
        rot = np.pad(np.copy(data_sfm.rot), (0, 1), 'constant')
        rot[3, 3] = 1
        return [np.copy(data_sfm.scale), np.copy(data_sfm.trans), transformations.quaternion_from_matrix(rot, isprecise=True)]

    def forward_img(self, index):
        data = self.anno[index]
        sfm_pose = self.sfm_pose(index)
        img = imread_rgb(self.image_path(index))
        mask = np.expand_dims(data.mask, 2)

        parts = data.parts.T.astype(float)
        kp = np.copy(parts)
        vis = kp[:, 2] > 0
        kp[vis, :2] -= 1

        bbox = self.crop_box(index)
        img, mask, kp, sfm_pose = self.crop_image(img, mask, bbox, kp, vis, sfm_pose)
        mirrored = self.is_train and (torch.randint(0, 2, size=(1,)).item() == 1)

        img_ref, mask_ref, kp_ref, pose_ref = self.scale_image(img.copy(), mask.copy(), kp.copy(), vis.copy(),
                                                               copy.deepcopy(sfm_pose), self.img_sizes[0])
        if mirrored:
            img_ref, mask_ref, kp_ref, pose_ref = self.mirror_image(img_ref, mask_ref, kp_ref, pose_ref)
        img_h, img_w = img_ref.shape[:2]
        kp_norm, pose_ref = self.normalize_kp(kp_ref, pose_ref, img_h, img_w)
        img_ref = np.transpose(img_ref, (2, 0, 1))

        extra_res = {}
        for res in self.img_sizes[1:]:
            img2, mask2, kp2, pose2 = self.scale_image(img.copy(), mask.copy(), kp.copy(), vis.copy(),
                                                       copy.deepcopy(sfm_pose), res)
            if mirrored:
                img2, mask2, kp2, pose2 = self.mirror_image(img2, mask2, kp2, pose2)
            extra_res[res] = (np.transpose(img2, (2, 0, 1)), mask2)
        return img_ref, kp_norm, mask_ref, pose_ref, mirrored, str(data.rel_path).replace('\\', '/'), extra_res

    @staticmethod
    def _normalize_pose(sfm_pose, img_h, img_w):
        sfm_pose[0] *= (1.0 / img_w + 1.0 / img_h)
        sfm_pose[1][0] = 2.0 * (sfm_pose[1][0] / img_w) - 1
        sfm_pose[1][1] = 2.0 * (sfm_pose[1][1] / img_h) - 1
        return sfm_pose

    def normalize_kp(self, kp, sfm_pose, img_h, img_w):
        vis = kp[:, 2, None] > 0
        new_kp = np.stack([2 * (kp[:, 0] / img_w) - 1, 2 * (kp[:, 1] / img_h) - 1, kp[:, 2]]).T
        return vis * new_kp, self._normalize_pose(sfm_pose, img_h, img_w)

    @staticmethod
    def _crop_pose(sfm_pose, bbox):
        sfm_pose[1][0] -= bbox[0]
        sfm_pose[1][1] -= bbox[1]
        return sfm_pose

    def crop_image(self, img, mask, bbox, kp, vis, sfm_pose):
        img = image_utils.crop(img, bbox, bgval=1)
        mask = image_utils.crop(mask, bbox, bgval=0)
        kp[vis, 0] -= bbox[0]
        kp[vis, 1] -= bbox[1]
        return img, mask, kp, self._crop_pose(sfm_pose, bbox)

    @staticmethod
    def _scale_pose(sfm_pose, scale):
        sfm_pose[0] *= scale
        sfm_pose[1] *= scale
        return sfm_pose

    def scale_image(self, img, mask, kp, vis, sfm_pose, img_size):
        scale = img_size / float(max(np.shape(img)[0], np.shape(img)[1]))
        img_scale, _ = image_utils.resize_img(img, scale)
        mask_scale, _ = image_utils.resize_img(mask, scale)
        kp[vis, :2] *= scale
        return img_scale, mask_scale, kp, self._scale_pose(sfm_pose, scale)

    @staticmethod
    def _mirror_pose(sfm_pose, width):
        R = transformations.quaternion_matrix(sfm_pose[2])
        sfm_pose[2] = transformations.quaternion_from_matrix(_MIRROR.dot(R.dot(_MIRROR)), isprecise=True)
        sfm_pose[1][0] = width - sfm_pose[1][0] - 1
        return sfm_pose

    def mirror_image(self, img, mask, kp, sfm_pose):
        img_flip = img[:, ::-1, :].copy()
        mask_flip = mask[:, ::-1].copy()
        new_x = img.shape[1] - kp[:, 0] - 1
        kp_flip = np.hstack((new_x[:, None], kp[:, 1:]))[self.kp_perm, :]
        return img_flip, mask_flip, kp_flip, self._mirror_pose(sfm_pose, img.shape[1])

    def __len__(self):
        return self.num_imgs

    def __getitem__(self, index):
        img, kp, mask, sfm_pose, mirrored, path, extra_res = self.forward_img(index)
        sfm_pose[0].shape = 1
        elem = {'img': img, 'kp': kp, 'mask': mask, 'sfm_pose': np.concatenate(sfm_pose), 'mirrored': mirrored,
                'inds': index, 'path': path}
        for res, img2 in extra_res.items():
            elem[f'img_{res}'] = img2
        return elem

    # ------------------------------------------------------------------------------------------------ device store
    def pose_row(self, index, mirrored):
        """float64 [7] (scale, tx, ty, q) of item index at img_sizes[0], as __getitem__ computes it, without the image."""
        bbox = self.crop_box(index)
        S = int(round(bbox[2])) - int(round(bbox[0])) + 1
        R = self.img_sizes[0]
        pose = self._scale_pose(self._crop_pose(self.sfm_pose(index), bbox), R / float(S))
        if mirrored:
            pose = self._mirror_pose(pose, R)
        pose = self._normalize_pose(pose, R, R)
        pose[0].shape = 1
        return np.concatenate(pose)

    def pose_table(self):
        """fp32 [N, 2, 8]: per item, unmirrored and mirrored (scale, tx, ty, 0, qw, qx, qy, qz), computed in float64 and
        rounded once (ImageDataset's FloatTensor conversions)."""
        t = np.zeros((len(self), 2, 8))
        for i in range(len(self)):
            for f in (0, 1):
                p = self.pose_row(i, f)
                t[i, f, :3], t[i, f, 4:] = p[:3], p[3:]
        return t.astype(np.float32)

    def windows(self):
        """int64 [N, 7]: per item the crop window inside the photo (ww, wh, wx0, wy0), the crop side S and the window's
        origin in the photo (x, y).  The photo size is the annotation mask's."""
        out = np.zeros((len(self), 7), np.int64)
        for i in range(len(self)):
            bbox = self.crop_box(i)
            im_h, im_w = self.anno[i].mask.shape
            x0, y0, wx0, wy0, ww, wh = image_utils.crop_window(bbox, im_h, im_w)
            out[i] = ww, wh, wx0, wy0, int(round(bbox[2])) - x0 + 1, x0 + wx0, y0 + wy0
        return out

    def packed_bytes(self):
        """Bytes of the packed photo store: 4 per window pixel (offsets, geometry and poses, 76 bytes per item, not
        counted)."""
        w = self.windows()
        return int((w[:, 0] * w[:, 1]).sum()) * 4

    def _window_words(self, i, win):
        ww, wh, _, _, _, px, py = (int(v) for v in win)
        rgb = imread_rgb_u8(self.image_path(i))
        mask = np.asarray(self.anno[i].mask)
        if rgb.shape[:2] != mask.shape:
            raise ValueError(f'{self.image_path(i)}: photo is {rgb.shape[1]}x{rgb.shape[0]}, its mask '
                             f'{mask.shape[1]}x{mask.shape[0]}')
        out = np.empty((wh, ww, 4), np.uint8)
        out[..., :3] = rgb[py:py + wh, px:px + ww]
        out[..., 3] = mask[py:py + wh, px:px + ww]
        return out.reshape(-1).view(np.int32)

    def to_device(self, device='cuda', workers=16, chunk=64):
        """Decode every photo once (`workers` threads, `chunk` photos at a time) and keep its crop window as RGBM words in
        one device buffer, with the offsets, window geometry and the pose table.  The store's size is checked against the
        free device memory first.  -> self."""
        import b3d
        import b3d.data
        device = torch.device(device)
        if device.type != 'cuda' or not torch.cuda.is_available():
            raise b3d.B3DError(f'to_device({device}): the packed store is read by a CUDA kernel and needs a CUDA device; '
                               'there is no CPU fallback')
        for r in self.img_sizes:
            if not 1 <= r <= b3d.data.MAX_SIDE:
                raise b3d.B3DError(f'to_device: image size {r} outside [1, {b3d.data.MAX_SIDE}]')
        if len(self.img_sizes) > b3d.data.MAX_RES:
            raise b3d.B3DError(f'to_device: at most {b3d.data.MAX_RES} image sizes, got {len(self.img_sizes)}')
        win = self.windows()
        if (win[:, 4] < 1).any():
            raise b3d.B3DError(f'to_device: item {int(np.argmin(win[:, 4]))} has an empty crop box')
        sizes = win[:, 0] * win[:, 1]
        need = int(sizes.sum()) * 4
        free, _ = torch.cuda.mem_get_info(device)
        if need > free:
            raise b3d.B3DError(f'to_device: the packed store needs {need} bytes, {free} are free on {device}')
        offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
        pixels = torch.empty(max(int(sizes.sum()), 1), dtype=torch.int32, device=device)
        n = len(self)
        with ThreadPoolExecutor(max_workers=workers) as pool:
            for a in range(0, n, chunk):
                ids = range(a, min(a + chunk, n))
                words = np.concatenate(list(pool.map(lambda i: self._window_words(i, win[i]), ids)))
                start = int(offsets[a])
                pixels[start:start + len(words)].copy_(torch.from_numpy(words))
        self.store = {'pixels': pixels, 'offsets': torch.from_numpy(offsets).to(device),
                      'geometry': torch.from_numpy(win[:, :5].astype(np.int32)).to(device),
                      'poses': torch.from_numpy(self.pose_table()).to(device),
                      'arange': torch.arange(n, dtype=torch.int32, device=device)}
        self.store_device = device
        torch.cuda.synchronize(device)
        return self

    def _require_store(self):
        if self.store is None:
            raise RuntimeError('call to_device() first')
        return self.store

    def batch_outputs(self, batch_size):
        """Fresh output tensors of one batch, in ImageDataset's order: X [B,4,R0,R0], [B,3,Rk,Rk] per extra size,
        scale [B,1], translation [B,3], rot [B,4], ind int64 [B]."""
        self._require_store()
        dev, B = self.store_device, batch_size
        imgs = [torch.empty(B, 4 if k == 0 else 3, r, r, device=dev) for k, r in enumerate(self.img_sizes)]
        return (*imgs, torch.empty(B, 1, device=dev), torch.empty(B, 3, device=dev), torch.empty(B, 4, device=dev),
                torch.empty(B, dtype=torch.int64, device=dev))

    def _gather(self, idx, flip, out):
        from b3d.data import image_batch
        st = self.store
        k = len(self.img_sizes)
        image_batch(st['pixels'], st['offsets'], st['geometry'], st['poses'], idx, flip, list(out[:k]), *out[k:])
        return out

    def gather(self, idx, flip=None, out=None):
        """The batch of items idx (int32 CUDA [B]) mirrored where flip (uint8 CUDA [B] or None) is set, written into
        `out` (static tensors from batch_outputs() for CUDA-graph capture: copy the step's indices into a static idx /
        flip device-to-device before replay) or into fresh tensors.  Outside a capture the indices are range-checked first
        (one synchronisation); inside one, an out-of-range index yields NaN rows (ind -1)."""
        import b3d
        self._require_store()
        if not torch.cuda.is_current_stream_capturing() and idx.numel():
            lo, hi = int(idx.min()), int(idx.max())
            if lo < 0 or hi >= len(self):
                raise b3d.B3DError(f'gather: index range [{lo}, {hi}] outside the {len(self)} items')
        return self._gather(idx, flip, out if out is not None else self.batch_outputs(idx.shape[0]))

    def train_batches(self, batch_size, epoch, seed=0, rank=0, world=1):
        """The epoch's batches of run_reconstruction.py's shuffled training loader, as ReconTrainer.step's tuples
        (X_real, gt_scale, gt_translation, gt_rot, gt_idx [B]) (extra images after X_real with a list img_size): order
        from epoch_order, the last partial batch kept (the loader has no drop_last), flips from epoch_flips when is_train.
        The order and flips are uploaded once; each batch is one b3d_image_batch launch."""
        self._require_store()
        order = epoch_order(len(self), epoch, seed, rank, world)
        dev = self.store_device
        idx = order.to(torch.int32).to(dev)
        flips = epoch_flips(len(order), epoch, seed, rank).to(dev) if self.is_train else None
        for a in range(0, len(order), batch_size):
            s = slice(a, min(a + batch_size, len(order)))
            yield self._gather(idx[s], flips[s] if flips is not None else None, self.batch_outputs(s.stop - a))

    def eval_batches(self, batch_size, rank=0, world=1):
        """Sequential, never mirrored batches over rank's contiguous shard (eval_shard), last batch ragged: the validation
        loader's (X_real, scale, translation, rot, ind), or with a list img_size the pseudo-GT loader's
        (X_R0, img_R1, ..., scale, translation, rot, ind)."""
        st = self._require_store()
        start, end = eval_shard(len(self), rank, world)
        for a in range(start, end, batch_size):
            b = min(a + batch_size, end)
            yield self._gather(st['arange'][a:b], None, self.batch_outputs(b - a))
