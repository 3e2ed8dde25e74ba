"""Drop-in for /root/reference/code/utils/inception.py (InceptionV3 :7-141): the Inception-v3 feature extractor behind the
FID evaluation (SURVEY §8f rank 4).  The reference wraps torchvision's `inception_v3(pretrained=True)` and returns the
activations of up to four blocks (64 / 192 / 768 / 2048 channels).

Here the network is written out (torchvision is not a dependency) with the SAME module tree, so a state dict of the
reference's wrapper loads with strict=True — `blocks.0.0.conv.weight`, `blocks.2.3.branch3x3dbl_2.bn.running_var`, ... —
and `load_torchvision_state_dict` takes torchvision's own `inception_v3_google-*.pth` (keys `Conv2d_1a_3x3.conv.weight`,
`Mixed_5b.branch1x1.bn.weight`, ...; the classifier and the auxiliary head are dropped, as the reference never runs them).

Execution (inference only, like the reference: `requires_grad=False`, `.eval()`):
* every BasicConv2d (conv, no bias -> BatchNorm eps 1e-3 -> ReLU) is ONE launch of libb3d's wgmma implicit-GEMM kernel
  (b3d_conv2d_tf32): the batch norm is folded into the weights (rounded to the nearest tf32) and a bias, ReLU is the
  epilogue's leaky slope 0, zero padding is the TMA out-of-bounds fill in both directions, and every branch writes
  straight into its channel slice of the block's concatenated NHWC output (no torch.cat);
* `avg_pool2d(3, stride 1, pad 1)` + 1x1 conv (the `branch_pool` of Mixed_5/6/7) is a 3x3 conv with all nine taps
  = w / 9 (count_include_pad=True makes this exact in real arithmetic);
* channel counts that are not multiples of the 32-wide K slice (3, 48, 80) are zero-padded once in the weights;
* max pools, the input transform and the final average pool are csrc/fid_kernels.cu.
CUDA only: no CPU fallback (a CPU tensor raises B3DError)."""
import ctypes
import os

import torch
import torch.nn as nn

from b3d import B3DError, check, dev, lib, ptr, stream_ptr

_HUB_FILE = "inception_v3_google-0cc3c7bd.pth"        # what torchvision's pretrained=True downloads into the hub cache


def _ints(v):
    return (ctypes.c_int * len(v))(*v)


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def round_tf32(w):
    """Round fp32 values to the nearest tf32 (10 mantissa bits), ties away from zero — cvt.rna.tf32.f32, what the weight
    bank does for the GAN (the tf32 tensor-core inputs would otherwise be truncated)."""
    bits = w.contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32)


class BasicConv2d(nn.Module):
    """Parameter holder with torchvision's names (conv.weight, bn.*); run through InceptionV3._conv."""

    def __init__(self, cin, cout, kernel_size, stride=1, padding=0):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, kernel_size, stride=stride, padding=padding, bias=False)
        self.bn = nn.BatchNorm2d(cout, eps=0.001)


class InceptionA(nn.Module):
    def __init__(self, cin, pool_features):
        super().__init__()
        self.branch1x1 = BasicConv2d(cin, 64, 1)
        self.branch5x5_1 = BasicConv2d(cin, 48, 1)
        self.branch5x5_2 = BasicConv2d(48, 64, 5, padding=2)
        self.branch3x3dbl_1 = BasicConv2d(cin, 64, 1)
        self.branch3x3dbl_2 = BasicConv2d(64, 96, 3, padding=1)
        self.branch3x3dbl_3 = BasicConv2d(96, 96, 3, padding=1)
        self.branch_pool = BasicConv2d(cin, pool_features, 1)
    # concatenation order; a list = a chain whose last member lands in the output; '~' = preceded by the 3x3 average pool
    plan = (["branch1x1"], ["branch5x5_1", "branch5x5_2"], ["branch3x3dbl_1", "branch3x3dbl_2", "branch3x3dbl_3"], ["~branch_pool"])


class InceptionB(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.branch3x3 = BasicConv2d(cin, 384, 3, stride=2)
        self.branch3x3dbl_1 = BasicConv2d(cin, 64, 1)
        self.branch3x3dbl_2 = BasicConv2d(64, 96, 3, padding=1)
        self.branch3x3dbl_3 = BasicConv2d(96, 96, 3, stride=2)
    plan = (["branch3x3"], ["branch3x3dbl_1", "branch3x3dbl_2", "branch3x3dbl_3"], ["maxpool"])


class InceptionC(nn.Module):
    def __init__(self, cin, c7):
        super().__init__()
        self.branch1x1 = BasicConv2d(cin, 192, 1)
        self.branch7x7_1 = BasicConv2d(cin, c7, 1)
        self.branch7x7_2 = BasicConv2d(c7, c7, (1, 7), padding=(0, 3))
        self.branch7x7_3 = BasicConv2d(c7, 192, (7, 1), padding=(3, 0))
        self.branch7x7dbl_1 = BasicConv2d(cin, c7, 1)
        self.branch7x7dbl_2 = BasicConv2d(c7, c7, (7, 1), padding=(3, 0))
        self.branch7x7dbl_3 = BasicConv2d(c7, c7, (1, 7), padding=(0, 3))
        self.branch7x7dbl_4 = BasicConv2d(c7, c7, (7, 1), padding=(3, 0))
        self.branch7x7dbl_5 = BasicConv2d(c7, 192, (1, 7), padding=(0, 3))
        self.branch_pool = BasicConv2d(cin, 192, 1)
    plan = (["branch1x1"], ["branch7x7_1", "branch7x7_2", "branch7x7_3"],
            ["branch7x7dbl_1", "branch7x7dbl_2", "branch7x7dbl_3", "branch7x7dbl_4", "branch7x7dbl_5"], ["~branch_pool"])


class InceptionD(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.branch3x3_1 = BasicConv2d(cin, 192, 1)
        self.branch3x3_2 = BasicConv2d(192, 320, 3, stride=2)
        self.branch7x7x3_1 = BasicConv2d(cin, 192, 1)
        self.branch7x7x3_2 = BasicConv2d(192, 192, (1, 7), padding=(0, 3))
        self.branch7x7x3_3 = BasicConv2d(192, 192, (7, 1), padding=(3, 0))
        self.branch7x7x3_4 = BasicConv2d(192, 192, 3, stride=2)
    plan = (["branch3x3_1", "branch3x3_2"], ["branch7x7x3_1", "branch7x7x3_2", "branch7x7x3_3", "branch7x7x3_4"], ["maxpool"])


class InceptionE(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.branch1x1 = BasicConv2d(cin, 320, 1)
        self.branch3x3_1 = BasicConv2d(cin, 384, 1)
        self.branch3x3_2a = BasicConv2d(384, 384, (1, 3), padding=(0, 1))
        self.branch3x3_2b = BasicConv2d(384, 384, (3, 1), padding=(1, 0))
        self.branch3x3dbl_1 = BasicConv2d(cin, 448, 1)
        self.branch3x3dbl_2 = BasicConv2d(448, 384, 3, padding=1)
        self.branch3x3dbl_3a = BasicConv2d(384, 384, (1, 3), padding=(0, 1))
        self.branch3x3dbl_3b = BasicConv2d(384, 384, (3, 1), padding=(1, 0))
        self.branch_pool = BasicConv2d(cin, 192, 1)
    # a tuple at the end of a chain = siblings that read the same tensor and are concatenated in that order
    plan = (["branch1x1"], ["branch3x3_1", ("branch3x3_2a", "branch3x3_2b")],
            ["branch3x3dbl_1", "branch3x3dbl_2", ("branch3x3dbl_3a", "branch3x3dbl_3b")], ["~branch_pool"])


class _Folded:
    """One BasicConv2d ready for b3d_conv2d_tf32: tap-major weights [T][Cout'][Cin'] (batch norm folded, tf32-rounded),
    bias [Cout'], tap offsets.  Taps are listed column by column: the per-tap persistent kernel takes every geometry of
    this network (odd widths, 1x7 / 7x1, stride 2), which the tap-shifted kernel covers with its generic tiles."""
    __slots__ = ("wt", "bias", "dy", "dx", "ntaps", "stride", "kh", "kw", "ph", "pw", "cin", "cinp", "cout", "coutp")


def _fold(m, avg_fold, device):
    w = m.conv.weight.detach().to(device=device, dtype=torch.float32)
    bn = m.bn
    scale = bn.weight.detach().float().to(device) / torch.sqrt(bn.running_var.detach().float().to(device) + bn.eps)
    bias = bn.bias.detach().float().to(device) - bn.running_mean.detach().float().to(device) * scale
    w = w * scale[:, None, None, None]
    cout, cin, kh, kw = w.shape
    (ph, pw), (sh, sw) = _pair(m.conv.padding), _pair(m.conv.stride)
    if sh != sw:
        raise B3DError("inception: anisotropic stride")
    if avg_fold:                                  # avg_pool2d(3, 1, 1) then this 1x1 conv == 3x3 conv, every tap w / 9
        if (kh, kw, ph, pw, sh) != (1, 1, 0, 0, 1):
            raise B3DError("inception: the pooled branch must be a 1x1 convolution")
        w = (w / 9.0).expand(cout, cin, 3, 3)
        kh = kw = 3
        ph = pw = 1
    f = _Folded()
    f.kh, f.kw, f.ph, f.pw, f.stride, f.cin, f.cout = kh, kw, ph, pw, sh, cin, cout
    f.cinp, f.coutp = -(-cin // 32) * 32, -(-cout // 32) * 32
    taps = [(r, s) for s in range(kw) for r in range(kh)]
    wt = torch.zeros(len(taps), f.coutp, f.cinp, device=device, dtype=torch.float32)
    for t, (r, s) in enumerate(taps):
        wt[t, :cout, :cin] = w[:, :, r, s]
    f.wt = round_tf32(wt)
    f.bias = torch.zeros(f.coutp, device=device, dtype=torch.float32)
    f.bias[:cout] = bias
    f.ntaps = len(taps)
    f.dy, f.dx = _ints([r - ph for r, s in taps]), _ints([s - pw for r, s in taps])
    return f


class InceptionV3(nn.Module):
    """Inception-v3 feature maps (reference :7-141).  Same constructor arguments plus `weights`:
    'pretrained' (default; the reference's behaviour) loads torchvision's ImageNet weights from $B3D_INCEPTION_WEIGHTS or the
    torch hub cache (where torchvision's download would have put them) and raises if the file is not there — this code never
    downloads; a path loads that file (torchvision's or this wrapper's key names); None keeps the random initialisation
    (tests)."""

    DEFAULT_BLOCK_INDEX = 3
    BLOCK_INDEX_BY_DIM = {64: 0, 192: 1, 768: 2, 2048: 3}

    def __init__(self, output_blocks=(DEFAULT_BLOCK_INDEX,), resize_input=True, normalize_input=True, requires_grad=False,
                 weights="pretrained"):
        super().__init__()
        if requires_grad:
            raise B3DError("InceptionV3: inference only (the FID evaluation never differentiates through it)")
        self.resize_input = resize_input
        self.normalize_input = normalize_input
        self.output_blocks = sorted(output_blocks)
        self.last_needed_block = max(output_blocks)
        assert self.last_needed_block <= 3, 'Last possible results block index is 3'
        self.blocks = nn.ModuleList()
        self.blocks.append(nn.Sequential(BasicConv2d(3, 32, 3, stride=2), BasicConv2d(32, 32, 3), BasicConv2d(32, 64, 3, padding=1),
                                         nn.MaxPool2d(kernel_size=3, stride=2)))
        if self.last_needed_block >= 1:
            self.blocks.append(nn.Sequential(BasicConv2d(64, 80, 1), BasicConv2d(80, 192, 3), nn.MaxPool2d(kernel_size=3, stride=2)))
        if self.last_needed_block >= 2:
            self.blocks.append(nn.Sequential(InceptionA(192, 32), InceptionA(256, 64), InceptionA(288, 64), InceptionB(288),
                                             InceptionC(768, 128), InceptionC(768, 160), InceptionC(768, 160), InceptionC(768, 192)))
        if self.last_needed_block >= 3:
            self.blocks.append(nn.Sequential(InceptionD(768), InceptionE(1280), InceptionE(2048), nn.AdaptiveAvgPool2d(output_size=(1, 1))))
        for m in self.modules():                                     # torchvision's init: truncated normal (std 0.1), BN = identity
            if isinstance(m, nn.Conv2d):
                nn.init.trunc_normal_(m.weight, mean=0.0, std=0.1, a=-2, b=2)
        for p in self.parameters():
            p.requires_grad = False
        self._folded = {}
        self.eval()
        if weights is not None:
            self.load_pretrained(None if weights == "pretrained" else weights)

    # ------------------------------------------------------------------------------------------------ weights
    _TV_NAMES = (("Conv2d_1a_3x3", "blocks.0.0"), ("Conv2d_2a_3x3", "blocks.0.1"), ("Conv2d_2b_3x3", "blocks.0.2"),
                 ("Conv2d_3b_1x1", "blocks.1.0"), ("Conv2d_4a_3x3", "blocks.1.1"),
                 ("Mixed_5b", "blocks.2.0"), ("Mixed_5c", "blocks.2.1"), ("Mixed_5d", "blocks.2.2"), ("Mixed_6a", "blocks.2.3"),
                 ("Mixed_6b", "blocks.2.4"), ("Mixed_6c", "blocks.2.5"), ("Mixed_6d", "blocks.2.6"), ("Mixed_6e", "blocks.2.7"),
                 ("Mixed_7a", "blocks.3.0"), ("Mixed_7b", "blocks.3.1"), ("Mixed_7c", "blocks.3.2"))

    def load_torchvision_state_dict(self, sd):
        """torchvision.models.inception_v3 key names -> this module (fc.* and AuxLogits.* are not part of the extractor)."""
        own = self.state_dict()
        out = {}
        for k, v in sd.items():
            for tv, mine in self._TV_NAMES:
                if k.startswith(tv + "."):
                    nk = mine + k[len(tv):]
                    if nk in own:
                        out[nk] = v
                    break
        missing = [k for k in own if k not in out and not k.endswith("num_batches_tracked")]
        if missing:
            raise B3DError(f"inception weights: {len(missing)} tensors missing, e.g. {missing[:3]}")
        self.load_state_dict(out, strict=False)

    def load_pretrained(self, path=None):
        if path is None:
            cands = [os.environ.get("B3D_INCEPTION_WEIGHTS"), os.path.join(torch.hub.get_dir(), "checkpoints", _HUB_FILE)]
            path = next((c for c in cands if c and os.path.exists(c)), None)
            if path is None:
                raise FileNotFoundError(
                    f"InceptionV3(weights='pretrained'): {_HUB_FILE} is neither at $B3D_INCEPTION_WEIGHTS nor in the torch hub cache "
                    f"({cands[1]}); this code never downloads.  Pass weights=<path> or weights=None (random, tests only).")
        sd = torch.load(path, map_location="cpu")
        if any(k.startswith("blocks.") for k in sd):
            self.load_state_dict(sd, strict=True)
        else:
            self.load_torchvision_state_dict(sd)

    def load_state_dict(self, *args, **kwargs):
        self._folded = {}
        return super().load_state_dict(*args, **kwargs)

    def _apply(self, fn, *args, **kwargs):
        self._folded = {}
        return super()._apply(fn, *args, **kwargs)

    def train(self, mode=True):
        if mode:
            raise B3DError("InceptionV3: inference only (batch norms are folded into the convolutions)")
        return super().train(False)

    # ------------------------------------------------------------------------------------------------ execution
    def _rec(self, m, avg_fold, device):
        key = (id(m), avg_fold, device)
        rec = self._folded.get(key)
        if rec is None:
            rec = self._folded[key] = _fold(m, avg_fold, device)
        return rec

    def _conv(self, x, m, avg_fold=False, out=None, coff=0):
        """x [N,H,W,Cin'] NHWC -> relu(bn(conv(x))).  out / coff: write the real channels into out[..., coff:coff + Cout];
        otherwise a fresh [N,Ho,Wo,Cout'] tensor (channels beyond Cout are exact zeros: zero weights, zero bias)."""
        f = self._rec(m, avg_fold, x.device)
        N, H, W, C = x.shape
        if C != f.cinp:
            raise B3DError(f"inception: layer expects {f.cinp} (padded) input channels, got {C}")
        Ho, Wo = (H + 2 * f.ph - f.kh) // f.stride + 1, (W + 2 * f.pw - f.kw) // f.stride + 1
        if out is None:
            out, cout = torch.empty(N, Ho, Wo, f.coutp, device=x.device, dtype=torch.float32), f.coutp
        else:
            cout = f.cout
            if tuple(out.shape[:3]) != (N, Ho, Wo) or coff % 4 or coff + cout > out.shape[3]:
                raise B3DError("inception: bad output slice")
        optr = ctypes.c_void_p(out.data_ptr() + 4 * coff)
        check(lib.b3d_conv2d_tf32(ptr(x), ptr(f.wt), ptr(f.bias), optr, N, H, W, C, Ho, Wo, cout, f.ntaps, f.dy, f.dx, f.stride, f.stride,
                                  Ho, Wo, out.shape[3], 1, 1, 0, 0, 0.0, None, 0, None, 0, 0, None, stream_ptr(x)))
        return out

    def _maxpool(self, x, out=None, coff=0):
        N, H, W, C = x.shape
        Ho, Wo = (H - 3) // 2 + 1, (W - 3) // 2 + 1
        if out is None:
            out = torch.empty(N, Ho, Wo, C, device=x.device, dtype=torch.float32)
        optr = ctypes.c_void_p(out.data_ptr() + 4 * coff)
        check(lib.b3d_maxpool3x3s2_nhwc(ptr(x), N, H, W, C, optr, out.shape[3], stream_ptr(x)))
        return out

    def _width(self, blk, name):
        """Output channels of one plan entry's final member."""
        if isinstance(name, tuple):
            return sum(getattr(blk, n).conv.out_channels for n in name)
        return getattr(blk, name.lstrip("~")).conv.out_channels

    def _mixed(self, blk, x):
        """One Inception block: every branch of `blk.plan` into its channel slice of the concatenated output."""
        N, H, W, C = x.shape
        widths = [C if chain == ["maxpool"] else self._width(blk, chain[-1]) for chain in blk.plan]
        Ho, Wo = ((H - 3) // 2 + 1, (W - 3) // 2 + 1) if isinstance(blk, (InceptionB, InceptionD)) else (H, W)
        out = torch.empty(N, Ho, Wo, sum(widths), device=x.device, dtype=torch.float32)
        off = 0
        for chain, width in zip(blk.plan, widths):
            if chain == ["maxpool"]:
                self._maxpool(x, out, off)
            else:
                h = x
                for name in chain[:-1]:
                    h = self._conv(h, getattr(blk, name))
                last = chain[-1]
                if isinstance(last, tuple):
                    o = off
                    for n in last:
                        self._conv(h, getattr(blk, n), out=out, coff=o)
                        o += getattr(blk, n).conv.out_channels
                else:
                    self._conv(h, getattr(blk, last.lstrip("~")), avg_fold=last.startswith("~"), out=out, coff=off)
            off += width
        return out

    def _input(self, inp):
        """Resize (bilinear, align_corners=False) + 2x - 1 + NCHW planes -> NHWC with 32 channels (reference :123-131)."""
        x = dev(inp, "images")
        B, _, H, W = x.shape
        OH, OW = (299, 299) if self.resize_input else (H, W)
        h = torch.empty(B, OH, OW, 32, device=x.device, dtype=torch.float32)
        check(lib.b3d_inception_input(ptr(x), B, H, W, OH, OW, 32, int(bool(self.normalize_input)), ptr(h), stream_ptr(x)))
        return h

    def _meanpool(self, h):
        N, Hh, Ww, C = h.shape
        pooled = torch.empty(N, 1, 1, C, device=h.device, dtype=torch.float32)
        check(lib.b3d_mean_hw_nhwc(ptr(h), N, Hh * Ww, C, ptr(pooled), stream_ptr(h)))
        return pooled

    def forward(self, inp):
        """inp [B,3,H,W] in (0,1) -> list of the selected blocks' activations, logically NCHW (channels-last storage)."""
        if inp.dim() != 4 or inp.shape[1] != 3:
            raise B3DError(f"InceptionV3: images must be [B,3,H,W], got {tuple(inp.shape)}")
        h = self._input(inp)
        outp = []
        for idx, block in enumerate(self.blocks):
            for m in block:
                if isinstance(m, BasicConv2d):
                    h = self._conv(h, m)
                elif isinstance(m, nn.MaxPool2d):
                    h = self._maxpool(h)
                elif isinstance(m, nn.AdaptiveAvgPool2d):
                    h = self._meanpool(h)
                else:
                    h = self._mixed(m, h)
            if idx in self.output_blocks:
                outp.append(h.permute(0, 3, 1, 2))
            if idx == self.last_needed_block:
                break
        return outp
