"""The training iteration of /root/reference/code/run_reconstruction.py as an importable module (the reference keeps
it in a script with argparse, dataset loading and .cuda() at import time): `ReconTrainer.step` restates :409-445 —

    pred_tex, mesh_map = generator(X_real)                       models/reconstruction.py
    raw_vtx = mesh_template.get_vertex_positions(mesh_map)       rendering/mesh_template.py:125-149
    vtx = transform_vertices(raw_vtx, scale, translation, rot, idx)   run_reconstruction.py:237-252 (DatasetParams deltas, z0)
    image, alpha = mesh_template.forward_renderer(renderer, vtx, pred_tex)
    loss = MSE(cat(image, alpha), X_real) + mesh_regularization * flat_warmup * loss_flat(normals(raw_vtx))
    two Adams: network (lr) and DatasetParams (lr_dataset)        :333-357

with the flat-loss warm-up factor 10 -> 1 in steps of 0.1 (:356, :438-439) and the criterion of --loss (mse|l1)
(:347-352).  `ReconTrainer.evaluate` is the validation pass evaluate_all (:255-319) and `ReconTrainer.render_multiview`
its turntable render (:188-221); `train_epoch` the epoch loop with its learning-rate halving (:466-470) and
`save_checkpoint` / `load_checkpoint` the checkpoints (:359-382, :472-481).  CUDA path: wgmma convolutions (models.reconstruction), ONE fused vertex-pipeline launch
(b3d.vertex), tiled DIB-R rasteriser + fused shader, fused RGBA-MSE|L1 / IoU and flat-loss kernels.  One process per
GPU; under torch.distributed the batch is sharded per rank, the gradients are all-reduced (mean) and the network's BatchNorm layers synchronise their statistics (SyncBN — the
reference never ran this script multi-GPU; SURVEY §8e states the deviation that keeps N-GPU == 1-GPU on the same
global batch)."""
import types

import numpy as np
import torch
import torch.distributed as dist

import checkpoint_io
from checkpoint_io import load_optimizer_state_dict, optimizer_state_dict
from b3d.mesh import rgba_l1_iou, rgba_mse_iou
from models.reconstruction import DatasetParams, ReconstructionNetwork
from rendering.renderer import Renderer
from rendering.utils import qmul, qrot
from utils.losses import loss_flat


TURNTABLE_ANGLES = (0, 45, 90, 135, 180, 225, 270, 315)


def turntable_rotations(device):
    """The quaternions of run_reconstruction.py's eight turntable views (:188-221), fp32 [8,4]: a fixed tilt, then each
    angle of TURNTABLE_ANGLES, scaled by 0.8, about the vertical axis."""
    rad = -90 / 180 * np.pi
    q0 = torch.tensor([np.cos(-rad / 2), 0, 0, np.sin(-rad / 2)], dtype=torch.float32, device=device)
    rad = 110 / 180 * np.pi
    q1 = torch.tensor([np.cos(-rad / 2), 0, np.sin(-rad / 2), 0], dtype=torch.float32, device=device)
    q0 = qmul(q0, q1)
    rot = []
    for angle in TURNTABLE_ANGLES:
        rad = angle / 180 * np.pi * 0.8
        rot.append(qmul(q0, torch.tensor([np.cos(-rad / 2), 0, 0, np.sin(-rad / 2)], dtype=torch.float32, device=device)))
    return torch.stack(rot, dim=0)


def turntable_vertices(rot, raw):
    """Camera-space vertices of object-space vertices raw [N,V,3] seen from the views rot [N,4] (:209-211)."""
    vtx = qrot(rot, raw) * 0.9
    vtx[:, :, 1:] *= -1
    return vtx


def default_args(**kw):
    """run_reconstruction.py's argparse defaults (:37-65) for the fields the step and the epoch loop read."""
    a = dict(symmetric=True, texture_resolution=128, mesh_resolution=32, image_resolution=256, loss='mse',
             optimize_deltas=True, optimize_z0=False, mesh_regularization=0.00005, lr=0.0001, lr_dataset=0.0001,
             epochs=1000, lr_decay_every=250)
    a.update(kw)
    return types.SimpleNamespace(**a)


class ReconTrainer:
    # keep_last_images: forward_loss keeps the batch and its render in `last_images` (run_reconstruction.py's
    # training-image summaries, :321-323, :487-488); off by default, as it holds one batch of renders into the next step
    keep_last_images = False
    last_images = None

    def __init__(self, args, mesh_template, dataset_size, device='cuda', capturable=False):
        if args.loss not in ('mse', 'l1'):
            raise ValueError(f"ReconTrainer: loss={args.loss!r}; the reference's criteria are 'mse' and 'l1'")
        self.args, self.tpl = args, mesh_template
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        net = ReconstructionNetwork(symmetric=args.symmetric, texture_res=args.texture_resolution,
                                    mesh_res=args.mesh_resolution)
        if self.world > 1:
            from sync_batchnorm import convert_model
            net = convert_model(net)
        self.generator = net.to(device)
        self.renderer = Renderer(args.image_resolution, args.image_resolution)
        fused = torch.device(device).type == 'cuda'
        self.optimizer = torch.optim.Adam(self.generator.parameters(), lr=args.lr, capturable=capturable, fused=fused)
        self.dataset_params = self.optimizer_dataset = None
        if args.optimize_deltas or args.optimize_z0:
            self.dataset_params = DatasetParams(args, dataset_size).to(device)
            self.optimizer_dataset = torch.optim.Adam(self.dataset_params.parameters(), lr=args.lr_dataset,
                                                      capturable=capturable, fused=fused)
        # flat-loss warm-up (:356, :438-439) as a device scalar so that a captured step keeps counting
        self.flat_warmup = torch.full((), 10.0, device=device)
        self.epoch = self.total_it = 0

    def criterion(self, image_pred, alpha_pred, X_real):
        """criterion(X_fake, X_real) over [B,4,H,W] + mean IoU on alpha, in one fused kernel (:347-352, :429-436)."""
        fn = rgba_l1_iou if self.args.loss == 'l1' else rgba_mse_iou
        return fn(image_pred, alpha_pred, X_real)

    def forward_loss(self, X_real, gt_scale, gt_translation, gt_rot, gt_idx=None):
        """-> (loss, recon_loss, flat_loss, miou); differentiable."""
        a, dp = self.args, self.dataset_params
        pred_tex, mesh_map = self.generator(X_real)
        scale, trans, z0 = gt_scale, gt_translation, None
        if a.optimize_deltas:
            translation_delta, scale_delta = dp(gt_idx, 'deltas')
            scale, trans = gt_scale + scale_delta, gt_translation + translation_delta
        if a.optimize_z0:
            z0 = dp(gt_idx, 'z0')
        raw_vtx, vtx = self.tpl.vertices_and_pose(mesh_map, scale, trans, gt_rot, z0)
        image_pred, alpha_pred = self.tpl.forward_renderer(self.renderer, vtx, pred_tex)
        if self.keep_last_images:
            self.last_images = (X_real, image_pred.detach(), alpha_pred.detach())
        recon_loss, miou = self.criterion(image_pred, alpha_pred, X_real)
        flat_loss = loss_flat(self.tpl.mesh, self.tpl.compute_normals(raw_vtx))
        loss = recon_loss + (a.mesh_regularization * self.flat_warmup) * flat_loss
        return loss, recon_loss, flat_loss, miou

    def step(self, X_real, gt_scale, gt_translation, gt_rot, gt_idx=None):
        self.generator.train()
        self.optimizer.zero_grad(set_to_none=True)
        if self.optimizer_dataset is not None:
            self.optimizer_dataset.zero_grad(set_to_none=True)
        loss, recon_loss, flat_loss, miou = self.forward_loss(X_real, gt_scale, gt_translation, gt_rot, gt_idx)
        with torch.no_grad():
            self.flat_warmup.copy_((self.flat_warmup - 0.1).clamp(min=1.0))
        loss.backward()
        if self.world > 1:
            from gan_training import _allreduce_grads
            _allreduce_grads(list(self.generator.parameters()), self.world)
            if self.dataset_params is not None:
                _allreduce_grads(list(self.dataset_params.parameters()), self.world)
        self.optimizer.step()
        if self.optimizer_dataset is not None:
            self.optimizer_dataset.step()
        return loss.detach(), recon_loss.detach(), flat_loss.detach(), miou

    # ------------------------------------------------------------------------------------------------ the epoch layer
    def train_epoch(self, batches):
        """One epoch of run_reconstruction.py's training loop (:407-470): `step` on every batch (X_real, gt_scale,
        gt_translation, gt_rot, gt_idx [B]), then epoch += 1 and, every args.lr_decay_every (default 250) epochs, the
        network optimiser's learning rate is halved (the DatasetParams optimiser keeps its rate).  -> the per-iteration
        step outputs.  A CUDA graph captured from `step` keeps the learning rate it was captured with: capture it again
        after this changes the rate, and after load_checkpoint."""
        outs = []
        for b in batches:
            outs.append(self.step(*b))
            self.total_it += 1
        self.epoch += 1
        if self.epoch % getattr(self.args, 'lr_decay_every', 250) == 0:
            for group in self.optimizer.param_groups:
                group['lr'] *= 0.5
        return outs

    def checkpoint(self):
        """The dict run_reconstruction.py's save_checkpoint writes (:472-481), plus 'flat_warmup': the flat-loss warm-up
        factor (the reference does not store it, and ignores the extra key)."""
        dp, od = self.dataset_params, self.optimizer_dataset
        return {
            'optimizer': optimizer_state_dict(self.optimizer),
            'generator': self.generator.state_dict(),
            'optimizer_dataset_params': optimizer_state_dict(od) if od is not None else None,
            'dataset_params': dp.state_dict() if dp is not None else None,
            'epoch': self.epoch,
            'iteration': self.total_it,
            'args': dict(vars(self.args)),
            'flat_warmup': float(self.flat_warmup),
        }

    def save_checkpoint(self, path):
        """Write checkpoint() to path (rank 0 under torch.distributed, then a barrier)."""
        checkpoint_io.save(self.checkpoint(), path)

    def load_checkpoint(self, path, mode='resume'):
        """run_reconstruction.py:359-377, loaded onto this trainer's device.  Both modes load the network and the
        DatasetParams (a trainer without DatasetParams accepts only a file without them), and epoch / iteration when
        present.  mode 'resume' (--continue_train) also loads both optimisers and the flat-loss warm-up factor; a file
        without 'flat_warmup' (one the reference wrote) restarts it at 10, as the reference does.  mode 'evaluate'
        (--evaluate, --generate_pseudogt) loads nothing more.  Parameters and buffers are copied in place."""
        if mode not in ('resume', 'evaluate'):
            raise ValueError(f"load_checkpoint: mode={mode!r}; expected 'resume' or 'evaluate'")
        chk = checkpoint_io.load(path, self.flat_warmup.device)
        if 'epoch' in chk:
            self.epoch, self.total_it = chk['epoch'], chk['iteration']
        self.generator.load_state_dict(chk['generator'])
        if self.dataset_params is not None:
            self.dataset_params.load_state_dict(chk['dataset_params'])
        elif chk.get('dataset_params') is not None:
            raise AssertionError("the checkpoint has DatasetParams but this trainer optimises neither deltas nor z0")
        if mode == 'resume':
            load_optimizer_state_dict(self.optimizer, chk['optimizer'])
            if self.optimizer_dataset is not None:
                load_optimizer_state_dict(self.optimizer_dataset, chk['optimizer_dataset_params'])
            self.flat_warmup.fill_(chk.get('flat_warmup', 10.0))

    @torch.no_grad()
    def evaluate(self, batches, distributed=False, samples=None):
        """The validation pass evaluate_all (:255-319) without its TensorBoard images: every batch (X_real, gt_scale,
        gt_translation, gt_rot[, idx]) is posed with the DATASET-MEAN DatasetParams (transform_vertices(..., None), :274)
        and scored with the configured criterion, loss_flat and mean IoU.  -> dict(recon_loss, flat_loss, miou, N): the
        per-sample means over the N images, which the reference logs as
        '[TEST] recon_loss {:.5f}, flat_loss {:.5f}, mIoU {:.5f}, N {}'.  A batch whose predicted and target alpha are
        both empty has a NaN IoU, as in the reference.  The sums stay on the device in fp64 (one host sync at the end).
        distributed: every rank passes its shard; the sums are all-reduced before the division, so every rank returns the
        values of the whole set (eval-mode batch norm couples no samples).  samples: positions in the sequence of
        `batches` (run_reconstruction.py's debug_ids, :161, :172, :287-299) whose images to hand back: the result's
        'samples' holds 'real' and 'fake' ([k,4,H,W] on the device, in position order) and 'render', the
        render_multiview tiles of the first four."""
        a, dp = self.args, self.dataset_params
        picks = sorted(int(i) for i in samples) if samples is not None else None
        real, fake, render, pos = [], [], [], 0
        self.generator.eval()
        sums = torch.zeros(4, dtype=torch.float64, device=next(self.generator.parameters()).device)
        for X_real, gt_scale, gt_translation, gt_rot, *_ in batches:
            B = X_real.shape[0]
            pred_tex, mesh_map = self.generator(X_real)
            scale, trans, z0 = gt_scale, gt_translation, None
            if a.optimize_deltas:                   # means [1,3] / [1,1] broadcast over the batch
                translation_delta, scale_delta = dp(None, 'deltas')
                scale, trans = gt_scale + scale_delta, gt_translation + translation_delta
            if a.optimize_z0:
                z0 = dp(None, 'z0').expand(B, 1)
            raw_vtx, vtx = self.tpl.vertices_and_pose(mesh_map, scale, trans, gt_rot, z0)
            image_pred, alpha_pred = self.tpl.forward_renderer(self.renderer, vtx, pred_tex)
            recon_loss, miou = self.criterion(image_pred, alpha_pred, X_real)
            flat_loss = loss_flat(self.tpl.mesh, self.tpl.compute_normals(raw_vtx))
            sums += torch.stack((recon_loss.double(), flat_loss.double(), miou.double(), sums.new_ones(()))) * B
            if picks is not None:
                rows = [i - pos for i in picks if pos <= i < pos + B]
                if rows:
                    real.append(X_real[rows])
                    fake.append(torch.cat((image_pred, alpha_pred), dim=3).permute(0, 3, 1, 2)[rows])
                    for r in rows:
                        if len(render) < 4:
                            render.append(self.render_multiview(raw_vtx, pred_tex, r))
            pos += B
        if distributed:
            dist.all_reduce(sums, op=dist.ReduceOp.SUM)
        recon, flat, miou, n = sums.tolist()
        out = dict(recon_loss=recon / n, flat_loss=flat / n, miou=miou / n, N=int(n))
        if picks is not None:
            out['samples'] = dict(real=torch.cat(real) if real else None, fake=torch.cat(fake) if fake else None,
                                  render=render)
        return out

    @torch.no_grad()
    def render_multiview(self, raw_vtx, pred_tex, idx=0):
        """Sample `idx` (object-space vertices raw_vtx [B,V,3], texture pred_tex [B,3,T,T]) rendered from the reference's
        eight turntable views (:188-221) in one batch-8 render -> numpy [2R, 4R, 3] tile (rows of four views) in [0, 1]."""
        rot = turntable_rotations(raw_vtx.device)
        raw = raw_vtx[idx:idx + 1].expand(len(rot), -1, -1).contiguous()
        tex = pred_tex[idx:idx + 1].expand(len(rot), -1, -1, -1).contiguous()
        view, _ = self.tpl.forward_renderer(self.renderer, turntable_vertices(rot, raw), tex)
        R = view.shape[1]
        tile = view.view(2, 4, R, view.shape[2], 3).permute(0, 2, 1, 3, 4).reshape(2 * R, 4 * view.shape[2], 3)
        return (tile.cpu().numpy() + 1) / 2
