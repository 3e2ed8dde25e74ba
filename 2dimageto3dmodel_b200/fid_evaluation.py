"""The FID evaluation loop of /root/reference/code/main.py (`evaluate_fid` :188-412 and its set-up :149-185) as an
importable class (the reference keeps it in a script with argparse and dataset loading at import time) — SURVEY §8f rank 4.

Per evaluation batch (main.py:216-317): truncated noise (rejection sampling, :244-253) -> running-average generator in
inference mode -> `render_and_score` (:282-293): displacement map -> vertices -> pose -> 299 x 299 render -> Inception
pool features; with pseudo-ground-truth in the batch also the texture-only (real mesh + generated texture) and mesh-only
(generated mesh + real texture) renders.  Then mean / covariance of the features and the Frechet distance to the
real-image statistics (:343-357), optionally on a subset of the size of the validation split (:359-376).

What runs where: generator, vertex pipeline (ONE fused launch for get_vertex_positions + qrot / scale / translate / flip,
`MeshTemplate.vertices_and_pose`), rasteriser + shader, Inception and the feature statistics are libb3d kernels; the
activations stay on the GPU (`utils.fid.FIDStatistics`) — the reference copies every batch's features to the host and
concatenates them.  Only the D x D eigen-decompositions of the final distance are host numpy, as in the reference.

`select_best_checkpoint` is main.py's `--evaluate --which_epoch best` search (:787-834).
"""
import glob
import os
import re

import numpy as np
import torch

from rendering.renderer import Renderer
from utils.fid import FIDStatistics, calculate_frechet_distance, calculate_stats, forward_inception_features, init_inception


def truncated_noise(n, dim, sigma, generator=None):
    """main.py:244-253, 'Gaussian truncation trick': N(0,1) noise whose components beyond +-sigma are re-drawn (on the host,
    like the reference, so that a seeded evaluation draws the same numbers)."""
    noise = torch.randn(n, dim, generator=generator)
    while (noise.abs() > sigma).any():
        mask = noise.abs() > sigma
        noise[mask] = torch.randn(int(mask.sum()), generator=generator)
    return noise


def load_real_statistics(path, evaluation_res=299, expect_images=None):
    """The reference's cache format (main.py:170-174): stats_m [D], stats_s [D,D] stored as its lower triangle, num_images,
    resolution -> (mu, sigma, num_images)."""
    stats = np.load(path, allow_pickle=True)
    if int(stats['resolution']) != evaluation_res:
        raise ValueError('Resolution does not match')
    n = int(stats['num_images'])
    if expect_images is not None and n != expect_images:
        raise ValueError('Number of images does not match')
    s = stats['stats_s']
    return stats['stats_m'], s + np.triu(s.T, 1), n


def save_real_statistics(path, mu, sigma, num_images, evaluation_res=299):
    np.savez(path, stats_m=mu, stats_s=np.tril(sigma), num_images=num_images, resolution=evaluation_res)


class FIDEvaluator:
    """generator: the running-average Generator (models.gan) — called as generator(noise, c, caption, return_attention=True);
    mesh_template: rendering.mesh_template.MeshTemplate; inception: utils.inception.InceptionV3 or None (-> init_inception()).
    """

    def __init__(self, generator, mesh_template, inception=None, evaluation_res=299, latent_dim=64, truncation_sigma=1.0,
                 device="cuda"):
        self.generator = generator
        self.mesh_template = mesh_template
        self.device = torch.device(device)
        self.inception = (inception if inception is not None else init_inception()).to(self.device).eval()
        self.evaluation_res = evaluation_res          # 299: "Same as Inception input resolution" (main.py:156)
        self.renderer = Renderer(evaluation_res, evaluation_res)
        self.latent_dim, self.truncation_sigma = latent_dim, truncation_sigma
        self.dim = 2048 if 3 in self.inception.output_blocks else {0: 64, 1: 192, 2: 768}[self.inception.output_blocks[-1]]
        self.m_real = self.s_real = None              # training-set statistics (cached after the first evaluation)
        self.m_real_val = self.s_real_val = self.n_images_val = None

    # ------------------------------------------------------------------------------------------------ real statistics
    def set_real_statistics(self, mu, sigma, validation=False, num_images=None):
        if validation:
            self.m_real_val, self.s_real_val, self.n_images_val = mu, sigma, num_images
        else:
            self.m_real, self.s_real = mu, sigma

    def score_images(self, images, stats):
        """images [B,3,R,R] in (0,1) on the GPU -> features accumulated into `stats`; returns the features."""
        feat = forward_inception_features(self.inception, images)
        stats.update(feat)
        return feat

    # ------------------------------------------------------------------------------------------------ one render
    def render_and_score(self, mesh_map, texture, data, stats, features_out=None):
        """main.py:282-293.  -> rendered images [B,3,R,R] in (0,1)."""
        scale = data['scale'].reshape(-1, 1)
        _, vtx = self.mesh_template.vertices_and_pose(mesh_map, scale, data['translation'], data['rotation'])
        image_pred, _ = self.mesh_template.forward_renderer(self.renderer, vtx, texture)
        image_pred = image_pred.permute(0, 3, 1, 2) / 2 + 0.5
        feat = self.score_images(image_pred, stats)
        if features_out is not None:
            features_out.append(feat)
        return image_pred

    # ------------------------------------------------------------------------------------------------ the loop
    @torch.no_grad()
    def evaluate(self, eval_batches, fast=False, seed=None, keep_features=False, distributed=False, samples=None):
        """eval_batches: iterable of dicts like the reference's eval_loader yields — 'idx' [B], 'rotation' [B,4], 'scale' [B]
        or [B,1], 'translation' [B,3]; optional 'class' [B] or [B,1], 'image' [B,3,R,R] in (0,1) (needed while the real
        statistics are not set), 'texture' + 'mesh' (pseudo-ground-truth: enables the texture-only / mesh-only scores unless
        fast).  seed: main.py:223-227 (args.evaluate): reseeds the noise stream.  distributed: every rank passes ITS shard of
        the evaluation set; the feature sums are all-reduced (torch.distributed) before the distances, so all ranks return the
        scores of the whole set (the validation-subset scores need the individual features and stay per rank).  samples:
        dataset indices whose images to hand back, main.py's visualisation set (:196-202, :296-340): out['samples'] maps
        'fake', 'fake_tex', 'fake_mesh' and, with pseudo-ground-truth, 'real', 'real_tex', 'fake_texture_only',
        'fake_mesh_only' to device tensors ordered as `samples` lists the indices found in this rank's batches ('index':
        those indices); selecting them costs one synchronisation per batch.  Returns a dict of scores (+ the feature
        matrices with keep_features)."""
        self.generator.eval()
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        st = {k: FIDStatistics(self.dim, self.device) for k in ("combined", "texture_only", "mesh_only", "real")}
        feats = {k: [] for k in st} if (keep_features or (self.m_real_val is not None and not fast)) else None
        has_pseudogt = False
        picks = found = None
        if samples is not None:
            picks = torch.as_tensor(np.asarray(samples), dtype=torch.int64, device=self.device)
            found = {k: [] for k in ('index', 'fake', 'fake_mesh', 'fake_tex', 'real', 'real_tex', 'fake_texture_only',
                                     'fake_mesh_only')}
        for data in eval_batches:
            data = {k: (v.to(self.device) if isinstance(v, torch.Tensor) else v) for k, v in data.items()}
            has_pseudogt = 'texture' in data and not fast
            if self.m_real is None:
                if 'image' not in data:
                    raise ValueError("real-image statistics are not set and the batch has no 'image'")
                if data['image'].shape[2] != self.evaluation_res or data['image'].shape[3] != self.evaluation_res:
                    raise ValueError("real images must be rendered at the evaluation resolution")
                self.score_images(data['image'].float(), st["real"])
            c = data.get('class')
            B = data['rotation'].shape[0]
            noise = truncated_noise(B, self.latent_dim, self.truncation_sigma, gen).to(self.device)
            pred_tex, pred_mesh_map, _ = self.generator(noise, c, None, return_attention=True)
            fake = self.render_and_score(pred_mesh_map, pred_tex, data, st["combined"], feats["combined"] if feats else None)
            rows = None
            if picks is not None:
                rows = torch.isin(data['idx'], picks).nonzero().flatten()
                if rows.numel():
                    found['index'].append(data['idx'][rows])
                    for k, v in (('fake', fake), ('fake_mesh', pred_mesh_map), ('fake_tex', pred_tex)):
                        found[k].append(v[rows])
                    if has_pseudogt and 'image' in data:
                        found['real'].append(data['image'][rows])
                    if has_pseudogt:
                        found['real_tex'].append(data['texture'][rows])
                else:
                    rows = None
            if has_pseudogt:
                tex_only = self.render_and_score(data['mesh'], pred_tex, data, st["texture_only"],
                                                 feats["texture_only"] if feats else None)
                mesh_only = self.render_and_score(pred_mesh_map, data['texture'], data, st["mesh_only"],
                                                  feats["mesh_only"] if feats else None)
                if rows is not None:
                    found['fake_texture_only'].append(tex_only[rows])
                    found['fake_mesh_only'].append(mesh_only[rows])
        if distributed:
            for k in st:
                st[k].all_reduce()
        if self.m_real is None:
            self.m_real, self.s_real = st["real"].finalize()
        out = {}
        m1, s1 = st["combined"].finalize()
        out["fid"] = calculate_frechet_distance(m1, s1, self.m_real, self.s_real)
        if has_pseudogt:
            out["fid_texture_only"] = calculate_frechet_distance(*st["texture_only"].finalize(), self.m_real, self.s_real)
            out["fid_mesh_only"] = calculate_frechet_distance(*st["mesh_only"].finalize(), self.m_real, self.s_real)
        if self.m_real_val is not None and not fast:
            # main.py:359-376: as many generated images as the validation split has, drawn without replacement
            rng = np.random.RandomState(1234) if seed is not None else np.random
            n_gen = st["combined"].n
            if self.n_images_val > n_gen:
                raise ValueError('Not supported')
            idx = torch.as_tensor(rng.choice(n_gen, size=self.n_images_val, replace=False), device=self.device)
            for key, name in (("combined", "fid_val"), ("texture_only", "fid_texture_only_val"), ("mesh_only", "fid_mesh_only_val")):
                if feats[key]:
                    f = torch.cat(feats[key], dim=0)
                    out[name] = calculate_frechet_distance(*calculate_stats(f[idx]), self.m_real_val, self.s_real_val)
        if keep_features:
            out["features"] = {k: torch.cat(v, dim=0) for k, v in feats.items() if v}
        out["num_generated"] = st["combined"].n
        if found is not None:
            out["samples"] = ordered_samples(found, picks)
        return out


def ordered_samples(found, picks):
    """The collected visualisation rows, reordered from evaluation order to the order of `picks` (main.py:199, :330-340:
    argsort(argsort(indices)) on the sorted indices); the indices not found are left out."""
    if not found['index']:
        return {'index': picks[:0]}
    index = torch.cat(found['index'])
    pos = (index.unsqueeze(1) == picks.unsqueeze(0)).int().argmax(dim=1)    # position of each found index in picks
    order = torch.argsort(pos)
    return {k: torch.cat(v)[order] for k, v in found.items() if v}


def select_best_checkpoint(trainer, evaluator, checkpoint_dir, eval_batches, seed=None, distributed=False):
    """main.py:787-834: every checkpoint_<epoch>.pth in checkpoint_dir (a name that matches the glob
    checkpoint_[0-9]*.pth but not checkpoint_([0-9]+).pth raises ValueError) is loaded in 'evaluate' mode into trainer
    (a GANTrainer) and scored by evaluator.evaluate(fast=True), newest epoch first; a later-visited checkpoint replaces
    the best one only on a strictly smaller FID.  The best checkpoint is then loaded and evaluated in full.  evaluator
    must score trainer's running-average generator (FIDEvaluator(trainer.trainer.generator_running_avg, ...)): the
    loads copy into it in place.  seed and distributed are passed to every evaluate call (the reference seeds every
    evaluation with 1234 in this mode).  -> dict(fast_fid={epoch: fid} in visit order,
    paths={epoch: path}, best_path, scores)."""
    checkpoints = {}
    for path in sorted(glob.glob(os.path.join(checkpoint_dir, 'checkpoint_[0-9]*.pth'))):
        m = re.search('checkpoint_([0-9]+).pth', path)
        if not m:
            raise ValueError(f'Invalid path detected: {path}')
        checkpoints[int(m.group(1))] = path
    if not checkpoints:
        raise ValueError(f'no checkpoint_<epoch>.pth in {checkpoint_dir}')
    fast_fid, best_fid, best_path = {}, float('inf'), None
    for epoch, path in sorted(checkpoints.items())[::-1]:
        trainer.load_checkpoint(path, 'evaluate')
        fid = evaluator.evaluate(eval_batches, fast=True, seed=seed, distributed=distributed)['fid']
        fast_fid[epoch] = fid
        if fid < best_fid:
            best_fid, best_path = fid, path
    if best_path is None:
        raise ValueError(f'no finite fast FID among {sorted(checkpoints)}')
    trainer.load_checkpoint(best_path, 'evaluate')
    scores = evaluator.evaluate(eval_batches, seed=seed, distributed=distributed)
    return dict(fast_fid=fast_fid, paths=checkpoints, best_path=best_path, scores=scores)
