"""The GAN step logic of /root/reference/code/main.py as an importable module (the reference keeps it in a
script with argparse at import time): `ModelWrapper` (main.py:449-526: 'g' / 'd' / 'inference' modes, fake‖real
batching, per-discriminator weights) and `GANTrainer` (main.py:588-589 optimisers, :691-723 G/D alternation with
d_steps_per_g, mesh smoothness term, :431-447 running-average generator), its epoch loop (`train_epoch`: :738-747 linear
learning-rate decay) and checkpoints (:599-633 loading, :749-770 save_checkpoint).  One process per GPU; under
torch.distributed the gradients are all-reduced (mean) in flat buckets after backward and the generator's
batch-norm statistics synchronise inside sync_batchnorm."""
import math

import torch
import torch.distributed as dist
import torch.nn as nn

import checkpoint_io
from checkpoint_io import load_optimizer_state_dict, optimizer_state_dict
from models.gan import Generator, MultiScaleDiscriminator
from utils.losses import GANLoss, loss_flat


class ModelWrapper(nn.Module):
    def __init__(self, args, generator_instantiator, discriminator=None):
        super().__init__()
        self.args = args
        self.generator = generator_instantiator()
        self.generator_running_avg = generator_instantiator()
        self.generator_running_avg.load_state_dict(self.generator.state_dict())
        for p in self.generator_running_avg.parameters():
            p.requires_grad = False
        self.discriminator = discriminator
        self.criterion_gan = GANLoss(getattr(args, 'loss', 'hinge'))

    def forward(self, mode, X_tex, X_alpha, X_mesh=None, C=None, caption=None, noise=None):
        args = self.args
        if mode not in ('g', 'd', 'inference'):
            raise AssertionError(mode)
        if noise is None:
            noise = torch.randn((X_alpha.shape[0], args.latent_dim), device=X_alpha.device)
        # the texture discriminator weighs double when only two discriminators look at 512^2 textures (main.py:487-490)
        d_weight = [2, 1] if args.num_discriminators == 2 and args.texture_resolution >= 512 else None
        if mode == 'g':
            pred_tex, pred_mesh = self.generator(noise, C, caption)
            X_fake = torch.cat((pred_tex * X_alpha, X_alpha), dim=1)
            out, mask = self.discriminator(X_fake, pred_mesh, C, caption)
            return self.criterion_gan(out, True, for_discriminator=False, mask=mask, weight=d_weight), pred_tex, pred_mesh
        if mode == 'd':
            with torch.no_grad():
                pred_tex, pred_mesh = self.generator(noise, C, caption)
                X_fake = torch.cat((pred_tex * X_alpha, X_alpha), dim=1)
                X_real = torch.cat((X_tex, X_alpha), dim=1)
                if (X_mesh is None) != (pred_mesh is None):
                    raise AssertionError("mesh maps must be given exactly when the generator has a mesh head")
                X = torch.cat((X_fake, X_real), dim=0)
                CC = torch.cat((C, C), dim=0) if C is not None else None
                M = torch.cat((pred_mesh, X_mesh), dim=0) if pred_mesh is not None else None
            out, mask = self.discriminator(X, M, CC, caption)
            B = X_alpha.shape[0]
            fake, real = [o[:B] for o in out], [o[B:] for o in out]
            mf = [m[:B] if m is not None else None for m in mask]
            mr = [m[B:] if m is not None else None for m in mask]
            if mask[0] is None:
                mf = mr = None
            loss_fake = self.criterion_gan(fake, False, for_discriminator=True, mask=mf, weight=d_weight)
            loss_real = self.criterion_gan(real, True, for_discriminator=True, mask=mr, weight=d_weight)
            return loss_fake, loss_real, pred_tex, pred_mesh
        with torch.no_grad():
            return self.generator_running_avg(noise, C, caption, return_attention=True)


def _allreduce_grads(params, world):
    """Mean all-reduce of the gradients (NCCL over NVLink): one flat bucket per ~64 MB; pack / unpack with multi-tensor
    (foreach) kernels — a handful of launches whatever the number of parameters."""
    grads = [p.grad for p in params if p.grad is not None]
    if not grads:
        return
    bucket, size = [], 0
    for g in grads + [None]:
        if g is not None:
            bucket.append(g)
            size += g.numel()
        if bucket and (g is None or size >= (1 << 24)):
            flat = torch.cat([b.reshape(-1) for b in bucket])
            dist.all_reduce(flat)
            flat.div_(world)
            views, off = [], 0
            for b in bucket:
                views.append(flat[off:off + b.numel()].view_as(b))
                off += b.numel()
            torch._foreach_copy_(bucket, views)
            bucket, size = [], 0


def allreduce_network_grads(net, world):
    """Gradient all-reduce of one network.  The convolution weights (>= 85 % of the parameters) already have their
    gradients in ONE flat buffer — the WeightBank's backward writes them there and autograd hands the parameters views of
    it — so that buffer is all-reduced in place (NCCL AVG: no pack, no divide, no unpack); the remaining small
    parameters (linear layers, embeddings, biases) go through one packed bucket."""
    params = [p for p in net.parameters() if p.grad is not None]
    bank = net.__dict__.get('_bank') if hasattr(net, '__dict__') else None
    flat = getattr(bank, 'last_dw', None) if bank else None
    done = set()
    if flat is not None and dist.get_backend() == 'nccl':
        base = flat.data_ptr()
        bp = bank.params()
        if all(p.grad is not None and p.grad.data_ptr() == base + 4 * sp['dw_off'] for p, sp in zip(bp, bank.specs)):
            dist.all_reduce(flat, op=dist.ReduceOp.AVG)
            done = {id(p) for p in bp}
    _allreduce_grads([p for p in params if id(p) not in done], world)


class GANTrainer:
    """One training iteration of main.py:672-736 per `step()` call: iteration k is a generator step when
    k % (1 + d_steps_per_g) == 0, else a discriminator step."""

    def __init__(self, args, mesh_template=None, device='cuda', capturable=False):
        self.args = args
        self.mesh_template = mesh_template
        use_mesh = not args.texture_only
        self.trainer = ModelWrapper(
            args, lambda: Generator(args, args.latent_dim, symmetric=getattr(args, 'symmetric_g', True), mesh_head=use_mesh),
            MultiScaleDiscriminator(args, 4)).to(device)
        g, d = self.trainer.generator, self.trainer.discriminator
        # betas=(0, 0.9) of main.py:588-589 (written as floats: the int 0 raises on torch >= 2, SURVEY App. A D14)
        # same update rule; on CUDA the multi-tensor "fused" implementation is one kernel per step instead of ~10
        fused = torch.device(device).type == 'cuda'
        self.optimizer_g = torch.optim.Adam(g.parameters(), lr=args.lr_g, betas=(0.0, 0.9), capturable=capturable, fused=fused)
        self.optimizer_d = torch.optim.Adam(d.parameters(), lr=args.lr_d, betas=(0.0, 0.9), capturable=capturable, fused=fused)
        self.total_it = 0
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.epoch = 0
        # main.py:591-594: the loss curves start with [0]; train_epoch appends one value per G / D iteration
        self.g_curve, self.d_fake_curve, self.d_real_curve, self.flat_curve = [0], [0], [0], [0]

    def update_generator_running_avg(self, epoch=1000):
        a = self.args.g_running_average_alpha
        alpha = math.pow(a, 100) if epoch < 10 else math.pow(a, 10) if epoch < 100 else a
        with torch.no_grad():
            src = self.trainer.generator.state_dict()
            fl_dst, fl_src = [], []
            for k, v in self.trainer.generator_running_avg.state_dict().items():
                if torch.is_floating_point(v):
                    fl_dst.append(v)
                    fl_src.append(src[k])
                else:
                    v.copy_(src[k])
            torch._foreach_mul_(fl_dst, alpha)
            torch._foreach_add_(fl_dst, fl_src, alpha=1 - alpha)

    def _freeze_discriminator(self, frozen):
        for p in self.trainer.discriminator.parameters():
            p.requires_grad_(not frozen)

    def g_step(self, X_alpha, C, noise=None, epoch=1000):
        self.optimizer_g.zero_grad(set_to_none=True)
        # The reference back-propagates the generator loss into the discriminator's weights as well and throws those
        # gradients away (optimizer_d.zero_grad() precedes every D step, main.py:717).  Freezing D here skips that
        # wasted weight-gradient work; the gradient that reaches the generator is unchanged.
        self._freeze_discriminator(True)
        try:
            loss, pred_tex, pred_mesh = self.trainer('g', None, X_alpha, None, C, None, noise)
        finally:
            self._freeze_discriminator(False)
        loss_gan = loss.mean()
        total, flat = loss_gan, None
        if pred_mesh is not None and self.mesh_template is not None:
            vtx = self.mesh_template.get_vertex_positions(pred_mesh)
            flat = loss_flat(self.mesh_template.mesh, self.mesh_template.compute_normals(vtx))
            total = total + self.args.mesh_regularization * flat
        # the step's loss terms, still on the device, for the curves train_epoch keeps (read once per epoch)
        self.last_terms = (loss_gan.detach(), flat.detach() if flat is not None else None)
        total.backward()
        if self.world > 1:
            allreduce_network_grads(self.trainer.generator, self.world)
        self.optimizer_g.step()
        self.update_generator_running_avg(epoch)
        return loss_gan.detach()

    def d_step(self, X_tex, X_alpha, X_mesh, C, noise=None):
        self.optimizer_d.zero_grad(set_to_none=True)
        loss_fake, loss_real, _, _ = self.trainer('d', X_tex, X_alpha, X_mesh, C, None, noise)
        loss_fake, loss_real = loss_fake.mean(), loss_real.mean()
        loss = loss_fake + loss_real
        self.last_terms = (loss_fake.detach(), loss_real.detach())
        loss.backward()
        if self.world > 1:
            allreduce_network_grads(self.trainer.discriminator, self.world)
        self.optimizer_d.step()
        return loss.detach()

    def step(self, X_tex, X_alpha, X_mesh, C, noise=None, epoch=1000):
        """epoch drives the warm-up of the running-average generator (main.py:431-438: alpha^100 for epoch < 10,
        alpha^10 for epoch < 100)."""
        is_g = self.total_it % (1 + self.args.d_steps_per_g) == 0
        out = self.g_step(X_alpha, C, noise, epoch) if is_g else self.d_step(X_tex, X_alpha, X_mesh, C, noise)
        self.total_it += 1
        return out

    # ------------------------------------------------------------------------------------------------ the epoch layer
    def train_epoch(self, batches):
        """One epoch of main.py's training loop (:672-747): `step` on every batch (a dict of step's arguments X_tex,
        X_alpha, X_mesh, C and optionally noise) at this trainer's `epoch`, then epoch += 1 and the linear learning-rate
        decay of both optimisers once epoch >= args.lr_decay_after (default 1000) while epoch < args.epochs (default 600).
        The loss curves get this epoch's values with one host synchronisation.  -> the per-iteration step outputs.
        A CUDA graph captured from `step` keeps the learning rate it was captured with: capture it again after this
        changes the rate, and after load_checkpoint."""
        outs, g, flat, d_fake, d_real = [], [], [], [], []
        for b in batches:
            is_g = self.total_it % (1 + self.args.d_steps_per_g) == 0
            outs.append(self.step(**b, epoch=self.epoch))
            if is_g:
                g.append(self.last_terms[0])
                if self.last_terms[1] is not None:
                    flat.append(self.last_terms[1])
            else:
                d_fake.append(self.last_terms[0])
                d_real.append(self.last_terms[1])
        vals = torch.stack(g + flat + d_fake + d_real).tolist() if outs else []
        for curve, n in ((self.g_curve, len(g)), (self.flat_curve, len(flat)), (self.d_fake_curve, len(d_fake)),
                         (self.d_real_curve, len(d_real))):
            curve.extend(vals[:n])
            vals = vals[n:]
        self.epoch += 1
        a = self.args
        after, epochs = getattr(a, 'lr_decay_after', 1000), getattr(a, 'epochs', 600)
        if after <= self.epoch < epochs:
            factor = 1 - min(max((self.epoch - after) / (epochs - after), 0), 1)
            for group in self.optimizer_g.param_groups:
                group['lr'] = a.lr_g * factor
            for group in self.optimizer_d.param_groups:
                group['lr'] = a.lr_d * factor
        return outs

    def checkpoint(self):
        """The dict main.py's save_checkpoint writes (:749-770): same keys, nesting and value types."""
        t = self.trainer
        return {
            'optimizer_g': optimizer_state_dict(self.optimizer_g),
            'optimizer_d': optimizer_state_dict(self.optimizer_d),
            'generator': t.generator.state_dict(),
            'generator_running_avg': t.generator_running_avg.state_dict(),
            'discriminator': t.discriminator.state_dict(),
            'epoch': self.epoch,
            'iteration': self.total_it,
            'g_curve': list(self.g_curve),
            'd_fake_curve': list(self.d_fake_curve),
            'd_real_curve': list(self.d_real_curve),
            'flat_curve': list(self.flat_curve),
            'args': dict(vars(self.args)),
        }

    def save_checkpoint(self, path):
        """Write checkpoint() to path (rank 0 under torch.distributed, then a barrier)."""
        checkpoint_io.save(self.checkpoint(), path)

    def load_checkpoint(self, path, mode='resume'):
        """main.py:599-633, loaded onto this trainer's device.  mode 'resume' (--continue_train): the networks, the
        running average, both optimisers, epoch, iteration (so the G / D alternation continues in phase) and the curves.
        mode 'evaluate' (--evaluate): generator_running_avg, plus generator / epoch / iteration / curves when the file
        has an 'epoch' (the shipped checkpoints hold generator_running_avg only).  Parameters and buffers are copied in
        place, so the weight banks keep their packed pointers and an FIDEvaluator built on generator_running_avg
        evaluates the loaded weights."""
        if mode not in ('resume', 'evaluate'):
            raise ValueError(f"load_checkpoint: mode={mode!r}; expected 'resume' or 'evaluate'")
        t = self.trainer
        chk = checkpoint_io.load(path, next(t.generator_running_avg.parameters()).device)
        if 'epoch' in chk:
            self.epoch, self.total_it = chk['epoch'], chk['iteration']
            self.g_curve, self.d_fake_curve = list(chk['g_curve']), list(chk['d_fake_curve'])
            self.d_real_curve, self.flat_curve = list(chk['d_real_curve']), list(chk['flat_curve'])
            t.generator.load_state_dict(chk['generator'])
        t.generator_running_avg.load_state_dict(chk['generator_running_avg'])
        if mode == 'resume':
            load_optimizer_state_dict(self.optimizer_g, chk['optimizer_g'])
            t.discriminator.load_state_dict(chk['discriminator'])
            load_optimizer_state_dict(self.optimizer_d, chk['optimizer_d'])
