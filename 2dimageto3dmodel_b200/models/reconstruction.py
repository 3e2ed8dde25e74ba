"""Drop-in for /root/reference/code/models/reconstruction.py: the image -> (texture, displacement map) network that
run_reconstruction.py trains through the renderer (SURVEY.md §8b, cfg4), and the per-image pose offsets.

Module tree, parameter and buffer names equal the reference's (`conv1e.weight`, `bn1e.running_mean`, `blk1.conv1.weight`,
`blk4_mesh.shortcut.weight`, `conv_tex.bias`, `fc1_tex.weight`, ... — its checkpoints load with strict=True) and modules
are created in the reference's order, so the same seed gives the same initial weights.  Every convolution is a
models.gan.TCConv2d, i.e. runs on libb3d's wgmma / TMA implicit-GEMM kernels (fprop, dgrad and wgrad, tf32 inputs, fp32
accumulate; the 3-channel 5x5 heads on the thin-head kernels).  The encoder's zero padding along x is materialised, along
y it is the TMA out-of-bounds fill; the decoder's replicate / circular x padding is explicit as in the reference.  Batch
norms, the three linear layers, nearest upsampling and tanh are stock torch ops on channels-last tensors.  CUDA only:
there is no CPU fallback (TCConv2d raises on CPU tensors).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from b3d.ew import CIRCULAR, REPLICATE, bn_act_pad, pad_x
from models.gan import TCConv2d
from rendering.utils import adjust_poles, symmetrize_texture

# encoder stages (reference :52-64): name suffix, channels in -> out, kernel, padding; all stride 2, no bias, BN + ReLU
_ENCODER = (("1e", 4, 64, 5, 2), ("2e", 64, 128, 3, 1), ("3e", 128, 256, 3, 1), ("4e", 256, 512, 3, 1), ("5e", 512, 64, 3, 1))
# decoder blocks in creation order (reference :77-99): attribute, channels in -> out, smallest texture_res that has it
_DECODER = (("blk1", 256, 512, 0), ("blk2", 512, 256, 0), ("blk3", 256, 256, 0), ("blk3b_tex", 256, 256, 128),
            ("blk3c_tex", 256, 256, 256), ("blk4_tex", 256, 128, 0), ("blk5_tex", 128, 64, 0))


class ResBlock(nn.Module):
    """conv3x3 -> BN -> ReLU -> conv3x3 -> BN -> ReLU, plus a 1x1 (or identity) shortcut (reference :7-26)."""

    def __init__(self, ch_in, ch_out, pad_fn):
        super().__init__()
        self.conv1 = TCConv2d(ch_in, ch_in, 3, padding=(1, 0), bias=False)
        self.conv2 = TCConv2d(ch_in, ch_out, 3, padding=(1, 0), bias=False)
        self.bn1, self.bn2 = nn.BatchNorm2d(ch_in), nn.BatchNorm2d(ch_out)
        self.relu = nn.ReLU(inplace=True)
        self.pad_fn = pad_fn
        self.shortcut = TCConv2d(ch_in, ch_out, 1, bias=False) if ch_in != ch_out else (lambda t: t)

    def forward(self, x):
        h = x
        for conv, bn in ((self.conv1, self.bn1), (self.conv2, self.bn2)):
            h = self.relu(bn(conv(self.pad_fn(h, 1))))
        return h + self.shortcut(x)

    def forward_fused(self, xp, up, pad_next, post_relu=False):
        """The same block on an input that is ALREADY replicate-padded by 1; returns the consumer's padded input
        pad(up([relu](h + skip)), pad_next).  Every conv output goes through ONE fused kernel (b3d.ew.bn_act_pad: batch
        norm + ReLU + residual + upsample + pad) instead of BN, ReLU, add, interpolate and pad passes."""
        a = bn_act_pad(self.conv1(xp), self.bn1, up=1, pad=1)
        y2 = self.conv2(a)
        if isinstance(self.shortcut, nn.Module):
            skip, off = self.shortcut(xp, x_crop=1), 0
        else:
            skip, off = xp, 1
        return bn_act_pad(y2, self.bn2, skip_nchw=skip, skip_off=off, up=up, pad=pad_next, post_relu=post_relu)


class ReconstructionNetwork(nn.Module):
    """RGBA image [B,4,256,256] -> (texture [B,3,R,R] in [-1,1], displacement map [B,3,32,32]) (reference :29-134).
    `symmetric=True` predicts one half of the UV map and mirrors it."""

    def __init__(self, symmetric=True, texture_res=64, mesh_res=32, interpolation_mode='nearest'):
        super().__init__()
        if mesh_res < 32 or texture_res not in (64, 128, 256):
            raise ValueError("mesh_res must be >= 32 and texture_res one of 64 / 128 / 256")
        if interpolation_mode not in ('nearest', 'bilinear'):
            raise ValueError(f"interpolation_mode={interpolation_mode!r}")
        self.symmetric, self.texture_res, self.interpolation_mode = symmetric, texture_res, interpolation_mode
        x_mode = REPLICATE if symmetric else CIRCULAR
        self.pad = lambda t, amount: pad_x(t, amount, x_mode)
        self.relu = nn.ReLU(inplace=True)
        up_kw = dict(mode='nearest') if interpolation_mode == 'nearest' else dict(mode='bilinear', align_corners=False)
        self.up = lambda t: F.interpolate(t, scale_factor=2, **up_kw)

        for tag, cin, cout, k, p in _ENCODER:                   # 256 -> 128 -> 64 -> 32 -> 16 -> 8
            setattr(self, "conv" + tag, TCConv2d(cin, cout, k, stride=2, padding=p, bias=False))
            setattr(self, "bn" + tag, nn.BatchNorm2d(cout))
        bottleneck = 256
        self.fc1e, self.bnfc1e = nn.Linear(64 * 8 * 8, bottleneck, bias=False), nn.BatchNorm1d(bottleneck)
        self.fc3e, self.bnfc3e = nn.Linear(bottleneck, 1024, bias=False), nn.BatchNorm1d(1024)

        self.base_res_h, self.base_res_w = 4, (2 if symmetric else 4)
        self.fc1_tex = nn.Linear(1024, self.base_res_h * self.base_res_w * 256)
        for name, cin, cout, min_res in _DECODER:
            if texture_res >= min_res:
                setattr(self, name, ResBlock(cin, cout, self.pad))
        self.conv_tex = TCConv2d(64, 3, 5, padding=(2, 0))

        # mesh head, zero-initialised so that training starts from the undeformed template (reference :101-103)
        self.blk4_mesh = ResBlock(256, 64, self.pad)
        self.conv_mesh = TCConv2d(64, 3, 5, padding=(2, 0))
        with torch.no_grad():
            self.conv_mesh.bias.zero_()
            self.conv_mesh.weight.zero_()
        print('Model parameters: {:.2f}M'.format(sum(p.nelement() for p in self.parameters()) / 1000000))

    def encode(self, image):
        h = image.contiguous(memory_format=torch.channels_last)
        for tag, *_ in _ENCODER:
            h = self.relu(getattr(self, "bn" + tag)(getattr(self, "conv" + tag)(h)))
        z = h.reshape(h.shape[0], -1)                           # (C, H, W) order, as the reference's .view on NCHW storage
        z = self.relu(self.bnfc1e(self.fc1e(z)))
        return self.relu(self.bnfc3e(self.fc3e(z)))

    def _decode_fused(self, h):
        """Decoder with the inter-convolution glue fused (replicate-padded tensors flow between the blocks)."""
        p = self.pad(h, 1)
        for name in ("blk1", "blk2", "blk3"):
            p = getattr(self, name).forward_fused(p, up=2, pad_next=1)
        shared = p                                              # 32 x 16 (+ pad): both heads branch from here
        for name in ("blk3b_tex", "blk3c_tex"):
            if hasattr(self, name):
                p = getattr(self, name).forward_fused(p, up=2, pad_next=1)
        t = self.blk4_tex.forward_fused(p, up=2, pad_next=1)
        t = self.blk5_tex.forward_fused(t, up=1, pad_next=2, post_relu=True)
        tex = torch.tanh(self.conv_tex(t))
        m = self.blk4_mesh.forward_fused(shared, up=1, pad_next=2, post_relu=True)
        mesh_map = adjust_poles(self.conv_mesh(m))
        return symmetrize_texture(tex), symmetrize_texture(mesh_map)

    def forward(self, x):
        z = self.encode(x)
        h = self.fc1_tex(z).view(z.shape[0], -1, self.base_res_h, self.base_res_w).contiguous(memory_format=torch.channels_last)
        if self.symmetric and self.interpolation_mode == 'nearest' and h.is_cuda and not getattr(self, 'disable_fusion', False):
            return self._decode_fused(h)
        for name in ("blk1", "blk2", "blk3"):
            h = self.up(getattr(self, name)(h))
        shared = h                                              # 32 x 16: both heads branch from here
        for name in ("blk3b_tex", "blk3c_tex"):
            if hasattr(self, name):
                h = self.up(getattr(self, name)(h))
        tex = self.blk5_tex(self.up(self.blk4_tex(h)))
        tex = torch.tanh(self.conv_tex(self.pad(self.relu(tex), 2)))
        mesh_map = adjust_poles(self.conv_mesh(self.pad(self.relu(self.blk4_mesh(shared)), 2)))
        if self.symmetric:
            tex, mesh_map = symmetrize_texture(tex), symmetrize_texture(mesh_map)
        return tex, mesh_map


class DatasetParams(nn.Module):
    """Learned per-image corrections of the estimated poses (reference :137-179): translation / scale deltas and the
    perspective parameter z0 = 1 + exp(theta).  Indices in [N, 2N) denote the mirrored copy of image i - N: its x
    translation changes sign.  `indices=None` returns the dataset mean (used at test time)."""

    def __init__(self, args, dataset_size):
        super().__init__()
        self.dataset_size = dataset_size
        if args.optimize_deltas:
            self.ds_translation = nn.Parameter(torch.zeros(dataset_size, 2))
            self.ds_scale = nn.Parameter(torch.zeros(dataset_size, 1))
        if args.optimize_z0:
            self.ds_z0 = nn.Parameter(torch.ones(dataset_size, 1))

    def forward(self, indices, mode):
        if mode not in ('deltas', 'z0'):
            raise ValueError(f"mode={mode!r}")
        x_sign = 1
        if indices is not None:
            x_sign = (1 - 2 * (indices // self.dataset_size).float()).unsqueeze(-1)
            indices = indices % self.dataset_size
        pick = (lambda p: p[indices]) if indices is not None else (lambda p: p.mean(dim=0, keepdim=True))
        if mode == 'z0':
            return 1 + torch.exp(pick(self.ds_z0))
        t = pick(self.ds_translation)
        translation_delta = torch.cat((t[:, :1] * x_sign, t[:, 1:2], torch.zeros_like(t[:, :1])), dim=1)
        return translation_delta, pick(self.ds_scale)
