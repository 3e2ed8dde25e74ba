"""The training iteration of /root/reference/code/run_reconstruction.py as an importable module (the reference keeps
it in a script with argparse, dataset loading and .cuda() at import time): `ReconTrainer.step` restates :409-445 —

    pred_tex, mesh_map = generator(X_real)                       models/reconstruction.py
    raw_vtx = mesh_template.get_vertex_positions(mesh_map)       rendering/mesh_template.py:125-149
    vtx = transform_vertices(raw_vtx, scale, translation, rot, idx)   run_reconstruction.py:237-252 (DatasetParams deltas, z0)
    image, alpha = mesh_template.forward_renderer(renderer, vtx, pred_tex)
    loss = MSE(cat(image, alpha), X_real) + mesh_regularization * flat_warmup * loss_flat(normals(raw_vtx))
    two Adams: network (lr) and DatasetParams (lr_dataset)        :333-357

with the flat-loss warm-up factor 10 -> 1 in steps of 0.1 (:356, :438-439).  CUDA path: wgmma convolutions
(models.reconstruction), ONE fused vertex-pipeline launch (b3d.vertex), tiled DIB-R rasteriser + fused shader, fused
RGBA-MSE / IoU and flat-loss kernels.  One process per GPU; under torch.distributed the batch is sharded per rank, the
gradients are all-reduced (mean) and the network's BatchNorm layers synchronise their statistics (SyncBN — the
reference never ran this script multi-GPU; SURVEY §8e states the deviation that keeps N-GPU == 1-GPU on the same
global batch)."""
import types

import torch
import torch.distributed as dist

from b3d.mesh import rgba_mse_iou
from models.reconstruction import DatasetParams, ReconstructionNetwork
from rendering.renderer import Renderer
from utils.losses import loss_flat


def default_args(**kw):
    """run_reconstruction.py's argparse defaults (:37-65) for the fields the step reads."""
    a = dict(symmetric=True, texture_resolution=128, mesh_resolution=32, image_resolution=256, loss='mse',
             optimize_deltas=True, optimize_z0=False, mesh_regularization=0.00005, lr=0.0001, lr_dataset=0.0001)
    a.update(kw)
    return types.SimpleNamespace(**a)


class ReconTrainer:
    def __init__(self, args, mesh_template, dataset_size, device='cuda', capturable=False):
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
        if args.loss != 'mse':
            raise ValueError("ReconTrainer: only the reference's default criterion (mse) is built on the fused loss kernel")
        # flat-loss warm-up (:356, :438-439) as a device scalar so that a captured step keeps counting
        self.flat_warmup = torch.full((), 10.0, device=device)

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
        recon_loss, miou = rgba_mse_iou(image_pred, alpha_pred, X_real)       # MSE over [B,4,H,W] + mean IoU on alpha
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
