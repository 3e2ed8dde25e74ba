"""The pseudo-ground-truth export of the reference's run_reconstruction.py (`--generate_pseudogt`, :499-658) as an
importable class: it turns a trained reconstruction model into the GAN stage's training data.

For every training photo (the pseudo-GT loader's batches (X_256, img_299, img_hd, scale, translation, rot, ind)):

    pred_tex, mesh_map = generator(X_256)                     eval mode; pred_tex resized to renderer_res // 8 if larger
    vtx = pose(mesh_map, scale + delta[ind], translation + delta[ind], rot, z0[ind])     MeshTemplate.vertices_and_pose
    unshaded render at renderer_res = max(1024, 2R)           b3d.mesh.render_indices
    texel visibility                                          b3d_texel_visibility (what d(render)/d(texture) > 0 marks)
    Inception features of img_299 / 2 + 0.5                   utils.fid.FIDStatistics (P3D: the car_imagenet subset)
    photo projected into UV space at R                        rendering.inverse_renderer.InverseRenderer
    mask, NCHW, fp16                                          b3d_pseudogt_pack, into one device staging buffer
    one copy to a pinned host slot per batch (two slots, CUDA events), records written by a thread pool

then poses_metadata.npz in index order and the real-image statistics precomputed_fid_299x299_train.npz (and, for CUB with
validation batches, _testval).  The records are byte-compatible with the reference's (data/pseudo_gt.py).

Deliberate differences from the reference: the statistics are written by fid_evaluation.save_real_statistics (fp64 lower
triangle, np.savez) instead of an fp32 triangle with savez_compressed (both load through load_real_statistics and the
reference's main.py:170-174); the Inception weights come from a local file (utils.fid.init_inception); the visibility is
computed from the render's index buffers instead of the full adjoint of the render.
"""
import os

import numpy as np
import torch
import torch.nn.functional as F

import b3d
from b3d.data import pseudogt_pack
from b3d.mesh import render_indices, texel_visibility
from data.pseudo_gt import pseudo_gt_dir, save_poses_metadata, save_pseudo_gt
from fid_evaluation import save_real_statistics
from rendering.inverse_renderer import InverseRenderer
from staging import Staging, byte_layout, views
from utils.fid import FIDStatistics, forward_inception_features, init_inception

INCEPTION_RES = 299


def renderer_resolution(pseudogt_resolution):
    """run_reconstruction.py:84: the visibility render is at least 1024 and at least twice the pseudo-GT resolution."""
    return max(1024, 2 * pseudogt_resolution)


def resize_texture(pred_tex, renderer_res):
    """:558-565: a texture larger than renderer_res // 8 is bilinearly resized to it (render >= 8x texture resolution keeps
    the visibility gradient free of aliasing)."""
    side = renderer_res // 8
    if pred_tex.shape[2] > side:
        return F.interpolate(pred_tex, size=(side, side), mode='bilinear', align_corners=False)
    return pred_tex


def imagenet_rows(paths):
    """:626-629: Pascal3D+'s real-image statistics use only the images of its ImageNet subset."""
    return [i for i, p in enumerate(paths) if p.startswith('car_imagenet')]


def _layout(B, C, R, img_shape, mesh_shape):
    """Byte offsets of one batch's fields in the staging buffer: fp16 texture / alpha / image, fp32 mesh map and pose rows
    (scale, tx, ty, tz, qw, qx, qy, qz), int64 indices; every field 16-byte aligned."""
    return byte_layout((('texture', torch.float16, (B, C, R, R)), ('texture_alpha', torch.float16, (B, 1, R, R)),
                        ('image', torch.float16, (B,) + tuple(img_shape)), ('mesh', torch.float32, (B,) + tuple(mesh_shape)),
                        ('pose', torch.float32, (B, 8)), ('ind', torch.int64, (B,))))


_views = views


def staged_records(views):
    """The records of one staged batch (the _layout views of a host slot): -> [(idx, record, pose row)].  Every tensor is a
    per-sample clone, so pickling a record writes that sample's planes only, never the whole slot."""
    out = []
    for i, idx in enumerate(views['ind'].tolist()):
        rec = {k: views[k][i].clone() for k in ('mesh', 'texture', 'texture_alpha', 'image')}
        out.append((idx, rec, views['pose'][i].clone()))
    return out


def write_poses_metadata(cache_dir, poses, paths):
    """poses_metadata.npz (:611-620) in index order: poses {idx: fp32 [8] (scale, tx, ty, tz, qw, qx, qy, qz)}, paths the
    dataset's per-index image paths.  -> the paths in the order written."""
    order = sorted(poses)
    table = torch.stack([poses[i] for i in order])
    ordered = [paths[i] for i in order]
    save_poses_metadata(cache_dir, table[:, :1].clone(), table[:, 1:4].clone(), table[:, 4:].clone(), ordered)
    return ordered


class PseudoGTExporter:
    """trainer: a ReconTrainer with the trained model loaded (load_checkpoint(path, 'evaluate')), or any object with its
    `generator`, `dataset_params` and `args` (optimize_deltas, optimize_z0); mesh_template: rendering.mesh_template.
    MeshTemplate; inception: utils.inception.InceptionV3 or None (-> init_inception(), local weights).  CUDA only."""

    def __init__(self, trainer, mesh_template, pseudogt_resolution=512, inception=None):
        if not torch.cuda.is_available():
            raise b3d.B3DError('PseudoGTExporter: the export runs on CUDA kernels and needs a CUDA device; there is no '
                               'CPU fallback')
        self.device = next(trainer.generator.parameters()).device
        if self.device.type != 'cuda':
            raise b3d.B3DError(f'PseudoGTExporter: the network is on {self.device}; move it to a CUDA device')
        self.trainer, self.tpl = trainer, mesh_template
        self.R = int(pseudogt_resolution)
        self.renderer_res = renderer_resolution(self.R)
        self.inverse_renderer = InverseRenderer(mesh_template.mesh, self.R, self.R)
        self.inception = (inception if inception is not None else init_inception()).to(self.device).eval()

    # ------------------------------------------------------------------------------------------------ one batch
    def _pose(self, mesh_map, scale, translation, rot, ind):
        """transform_vertices(raw_vtx, gt_scale, gt_translation, gt_rot, gt_idx) (:237-252) with the per-index deltas."""
        a, dp = self.trainer.args, self.trainer.dataset_params
        z0 = None
        if a.optimize_deltas:
            translation_delta, scale_delta = dp(ind, 'deltas')
            scale, translation = scale + scale_delta, translation + translation_delta
        if a.optimize_z0:
            z0 = dp(ind, 'z0')
        return self.tpl.vertices_and_pose(mesh_map, scale, translation, rot, z0)[1]

    def _reset(self):
        """Forget the buffers and statistics of a previous export (each export allocates its own once)."""
        self._bufs = self._vis = self._words = self._stats = None
        self._staging = Staging(self.device, 'export')

    def _buffers(self, B):
        """Render / visibility buffers for batches of up to B samples, allocated once per export."""
        if self._bufs is None or self._bufs[0].shape[0] < B:
            H = self.renderer_res
            d = self.device
            self._bufs = (torch.empty(B, H, H, device=d, dtype=torch.int32), torch.empty(B, H, H, 3, device=d),
                          torch.empty(B, H, H, 3, device=d), torch.empty(B, H, H, 1, device=d))
            self._vis = self._words = None
        return self._bufs

    @torch.no_grad()
    def _device_batch(self, batch, keep):
        """GPU work of one batch: fills the device staging buffer (allocated at the first batch, the largest) and returns
        the batch's byte layout and size."""
        X, img299, hd, scale, translation, rot, ind = (t.to(self.device) for t in batch)
        ind = ind.reshape(-1)
        B = X.shape[0]
        pred_tex, mesh_map = self.trainer.generator(X)
        pred_tex = resize_texture(pred_tex, self.renderer_res)
        vtx = self._pose(mesh_map, scale, translation, rot, ind)
        uvs, tex = self.tpl.adjust_uv_and_texture(pred_tex)
        Th, Tw = tex.shape[2], tex.shape[3]
        H = self.renderer_res
        imidx, imwei, fuv = render_indices(vtx, self.tpl.mesh.faces, uvs, self.tpl.mesh.face_textures, H, H,
                                           out=self._buffers(B))
        Tw_out = pred_tex.shape[3]
        if self._vis is None or self._vis.shape[0] < B or tuple(self._vis.shape[1:]) != (Th, Tw_out):
            self._vis = torch.empty(B, Th, Tw_out, device=self.device, dtype=torch.uint8)
            self._words = torch.empty(B, (Th * Tw_out + 31) // 32, device=self.device, dtype=torch.int32)
        vis = texel_visibility(imidx, imwei, fuv, Th, Tw, self.tpl.is_symmetric, out=self._vis, words=self._words)

        feat = forward_inception_features(self.inception, img299 / 2 + 0.5)
        if keep is not None:                 # rows outside the subset add exact zeros to the fp64 sums
            feat = feat * keep[ind].unsqueeze(1)
        if self._stats is None:
            self._stats = FIDStatistics(feat.shape[1], self.device)
        self._stats.update(feat)

        inv_tex, inv_alpha = self.inverse_renderer(vtx, hd)
        lay, nbytes = _layout(B, inv_tex.shape[3], self.R, img299.shape[1:], mesh_map.shape[1:])
        v = _views(self._staging.device_buffer(nbytes, B), lay)
        pseudogt_pack(vis, inv_tex.contiguous(), inv_alpha.contiguous(), img299.contiguous(), v['texture'],
                      v['texture_alpha'], v['image'])
        v['mesh'].copy_(mesh_map)
        v['pose'][:, :1].copy_(scale.reshape(B, 1))
        v['pose'][:, 1:4].copy_(translation)
        v['pose'][:, 4:].copy_(rot)
        v['ind'].copy_(ind)
        return lay, nbytes

    # ------------------------------------------------------------------------------------------------ the loop
    def export(self, batches, paths, cache_dir, dataset, val_batches=None, writers=8):
        """batches: the pseudo-GT loader's (X_256, img_299, img_hd, scale, translation, rot, ind) tuples on the device
        (cmr_data's `ds.to_device(); ds.eval_batches(B)` with img_size [256, 299, renderer_res]); paths: the dataset's
        per-index image paths (`ds.get_paths()`); cache_dir: cache/<dataset>; dataset: 'cub' or 'p3d'; val_batches: for
        CUB the 299^2 validation batches (X, ...) whose X[:, :3] / 2 + 0.5 gives the testval statistics; writers: threads
        that compress and write the records.  Every batch but the last must have the first batch's size.
        -> dict(records, num_images_train, num_images_testval, pseudogt_dir, poses_metadata, fid_train, fid_testval)."""
        if dataset not in ('cub', 'p3d'):
            raise ValueError(f"export: dataset={dataset!r}; expected 'cub' or 'p3d'")
        self.trainer.generator.eval()
        out_dir = pseudo_gt_dir(cache_dir, self.R)
        os.makedirs(out_dir, exist_ok=True)
        keep = None
        if dataset == 'p3d':
            keep = torch.zeros(len(paths), device=self.device)
            keep[imagenet_rows(paths)] = 1
        self._reset()
        poses = {}

        def device_batch(batch):
            lay, nbytes = self._device_batch(batch, keep)
            return lay, nbytes, lay['ind'][2][0]

        def drain(host, lay, submit):
            """Host side of one staged batch: clone every sample out of the pinned slot, queue the writes."""
            for idx, rec, pose in staged_records(_views(host, lay)):
                poses[idx] = pose
                submit(save_pseudo_gt, out_dir, idx, rec)

        self._staging.run(batches, device_batch, drain, writers)
        if not poses:
            raise ValueError('export: no batches')

        meta_paths = write_poses_metadata(cache_dir, poses, paths)
        stats = self._stats
        if dataset == 'p3d':                  # the zeroed rows outside the subset are not images of the statistics
            stats.n = len(imagenet_rows(meta_paths))
        n_train = stats.n
        out = dict(records=len(poses), num_images_train=n_train, num_images_testval=None, pseudogt_dir=out_dir,
                   poses_metadata=os.path.join(cache_dir, 'poses_metadata.npz'), fid_train=None, fid_testval=None)
        out['fid_train'] = self._save_stats(stats, cache_dir, 'train')
        if dataset == 'cub' and val_batches is not None:
            vstats = FIDStatistics(stats.dim, self.device)
            with torch.no_grad():
                for X, *_ in val_batches:
                    vstats.update(forward_inception_features(self.inception, X[:, :3] / 2 + 0.5))
            out['num_images_testval'] = vstats.n
            out['fid_testval'] = self._save_stats(vstats, cache_dir, 'testval')
        return out

    @staticmethod
    def _save_stats(stats, cache_dir, split):
        mu, sigma = stats.finalize()
        path = os.path.join(cache_dir, f'precomputed_fid_{INCEPTION_RES}x{INCEPTION_RES}_{split}.npz')
        save_real_statistics(path, mu, sigma, stats.n, INCEPTION_RES)
        return path
