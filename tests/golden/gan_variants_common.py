"""Shared recipe of the GAN-variant golden test: the generator / discriminator options beyond the default configuration
(norm_g instance / none, norm_d instance, the asymmetric full-width generator), built with the same seeds for the
reference (CPU) and the CUDA modules.  Inputs and the G / D steps are gan_common's."""
import torch

import gan_common as GC

B = 2
CONFIGS = {
    "cfg1": dict(res=256, nd=2, norm_g="instance", norm_d="none", symmetric=True),
    "cfg2": dict(res=256, nd=2, norm_g="none", norm_d="none", symmetric=True),
    "cfg3": dict(res=256, nd=2, norm_g="syncbatch", norm_d="instance", symmetric=True),
    "cfg4": dict(res=256, nd=2, norm_g="syncbatch", norm_d="none", symmetric=False),
    "cfg5": dict(res=512, nd=3, norm_g="instance", norm_d="instance", symmetric=False),
}


def make_args(name):
    cfg = CONFIGS[name]
    args = GC.make_args(cfg["res"], cfg["nd"])
    args.norm_g, args.norm_d = cfg["norm_g"], cfg["norm_d"]
    args.symmetric_g = cfg["symmetric"]
    return args


def build(gan_module, name, seed=123):
    """-> (args, G, D).  Same construction order and seeds as gan_common.build; the instance norms' affine weight / bias
    (ones / zeros at construction) are moved away from the identity so their gradients are exercised."""
    args = make_args(name)
    torch.manual_seed(seed)
    G = gan_module.Generator(args, 64, symmetric=args.symmetric_g, mesh_head=True)
    D = gan_module.MultiScaleDiscriminator(args, 4)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        G.conv_mesh.weight.copy_(torch.randn(G.conv_mesh.weight.shape, generator=g) * 0.02)
        G.conv_mesh.bias.copy_(torch.randn(G.conv_mesh.bias.shape, generator=g) * 0.02)
        for mname, m in sorted(D.named_modules(), key=lambda t: t[0]):
            if isinstance(m, torch.nn.InstanceNorm2d) and m.affine:
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) * 0.8 + 0.6)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.2)
    return args, G, D


def state_summary(module):
    """(names, shapes as strings, fp64 sums) of a module's state dict, in state-dict order."""
    sd = module.state_dict()
    names = list(sd.keys())
    shapes = ["x".join(str(s) for s in sd[n].shape) for n in names]
    sums = [float(sd[n].double().sum()) for n in names]
    return names, shapes, sums
