"""The generator's upsampled-input convolutions on the GPU (b3d.conv.conv2d_up2_banked and the glue around it).

  * every upsampled conv1 (+ its 1x1 shortcut) at its cfg3 shape (batch 32, 256^2) and its cfg5 shape (batch 8, 512^2):
    forward, the epilogue's BatchNorm statistics, input gradient and weight gradients from the bank against fp64
    F.interpolate + F.conv2d and autograd, within 4e-3 of the largest fp64 magnitude (test_workload_shapes_gpu.py's bound),
    in both x-padding modes;
  * the half-resolution residual of cbn_act_pad (skip_half) against the same glue on the upsampled skip, forward and
    gradients;
  * the fused generator on the bank (low-resolution maps between the blocks) against its module path, both pad modes:
    outputs, parameter gradients and running statistics within test_bank_gpu.py's bank-against-module bounds;
  * launch coverage: over one real cfg3 and one real cfg5 generator + discriminator step every call of the new launch
    helpers has a geometry of the table below, and no upsampled conv1 reaches the generic banked convolution."""
import sys
import types

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import gan_common as GC                  # noqa: E402

import b3d.conv as C                     # noqa: E402
from b3d.bank import WeightBank          # noqa: E402
from b3d.ew import CIRCULAR, REPLICATE, cbn_act_pad  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = 4e-3

# (config, layer, N, low-resolution H, W, Cin, Cout of conv1, Cout of the 1x1 shortcut or 0 = identity)
TABLE = [
    ("cfg3", "blk2", 32, 8, 4, 512, 256, 256), ("cfg3", "blk3a", 32, 16, 8, 256, 256, 0),
    ("cfg3", "blk3_mesh", 32, 16, 8, 256, 64, 64), ("cfg3", "blk4", 32, 32, 16, 256, 128, 128),
    ("cfg3", "blk5", 32, 64, 32, 128, 128, 0), ("cfg3", "blk6", 32, 128, 64, 128, 64, 64),
    ("cfg5", "blk2", 8, 8, 4, 512, 256, 256), ("cfg5", "blk3a", 8, 16, 8, 256, 256, 0),
    ("cfg5", "blk3b", 8, 32, 16, 256, 256, 0), ("cfg5", "blk3_mesh", 8, 16, 8, 256, 64, 64),
    ("cfg5", "blk4", 8, 64, 32, 256, 128, 128), ("cfg5", "blk5", 8, 128, 64, 128, 128, 0),
    ("cfg5", "blk6", 8, 256, 128, 128, 64, 64),
]


def _pad(x, mode):
    return torch.cat([x[..., :1], x, x[..., -1:]], -1) if mode == REPLICATE else torch.cat([x[..., -1:], x, x[..., :1]], -1)


def _close(a, ref, what):
    err, mag = float((a.double() - ref).abs().max()), float(ref.abs().max())
    assert err <= TOL * mag, f"{what}: |err| {err:.3e} > {TOL} * {mag:.3e}"


def _bank(Cin, Cout, Csc, seed):
    torch.manual_seed(seed)
    convs = {"conv1": nn.Conv2d(Cin, Cout, 3, bias=False)}
    if Csc:
        convs["shortcut"] = nn.Conv2d(Cin, Csc, 1, bias=False)
    for m in convs.values():
        m.to(DEV)
    return convs, WeightBank(convs, up2=["conv1"])


@pytest.mark.parametrize("mode", [REPLICATE, CIRCULAR])
@pytest.mark.parametrize("cfg,name,N,H,W,Cin,Cout,Csc", TABLE, ids=[f"{c}-{n}" for c, n, *_ in TABLE])
def test_layer(cfg, name, N, H, W, Cin, Cout, Csc, mode):
    convs, bank = _bank(Cin, Cout, Csc, N + H + Cin)
    x = torch.randn(N, Cin, H, W, device=DEV)
    xp = _pad(x, mode).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    lws = bank.forward(True)
    stats = torch.zeros(2 * Cout, device=DEV, dtype=torch.float64)
    y, sc = C.conv2d_up2_banked(xp, lws["conv1"], lws.get("shortcut"), stats=stats)
    gy = torch.randn_like(y)
    gsc = torch.randn_like(sc) if Csc else None
    torch.autograd.backward([y] + ([sc] if Csc else []), [gy] + ([gsc] if Csc else []))
    torch.cuda.synchronize()

    # fp64: the upsampled map, padded, convolved (pad columns of the upsampled map = Xp's pad columns)
    xd = xp.detach().double().requires_grad_(True)
    w1 = convs["conv1"].weight.detach().double().requires_grad_(True)
    u = F.interpolate(xd[..., 1:-1], scale_factor=2, mode="nearest")
    up = torch.cat([xd[..., :1].repeat_interleave(2, 2), u, xd[..., -1:].repeat_interleave(2, 2)], -1)
    ref = F.conv2d(up, w1, padding=(1, 0))
    _close(y, ref, "forward")
    _close(stats[:Cout], ref.sum((0, 2, 3)), "sum")
    _close(stats[Cout:], (ref * ref).sum((0, 2, 3)), "sum of squares")
    outs, grads = [ref], [gy.double()]
    if Csc:
        ws = convs["shortcut"].weight.detach().double().requires_grad_(True)
        rs = F.conv2d(xd[..., 1:-1], ws)
        _close(sc, rs, "shortcut forward")
        outs.append(rs)
        grads.append(gsc.double())
    params = [xd, w1] + ([ws] if Csc else [])
    gref = torch.autograd.grad(outs, params, grads)
    _close(xp.grad, gref[0], "input gradient")
    _close(convs["conv1"].weight.grad, gref[1], "conv1 weight gradient")
    if Csc:
        _close(convs["shortcut"].weight.grad, gref[2], "shortcut weight gradient")


@pytest.mark.parametrize("post_leaky", [False, True])
@pytest.mark.parametrize("mode", [REPLICATE, CIRCULAR])
def test_half_resolution_skip(mode, post_leaky):
    """cbn_act_pad(skip_half=True) == cbn_act_pad on the x2-upsampled skip, forward and all gradients."""
    from models.gan import ConditionalBatchNorm2d
    args = types.SimpleNamespace(norm_g="batch")
    torch.manual_seed(3)
    N, Cc, H, W = 4, 64, 16, 12
    cbn = ConditionalBatchNorm2d(args, Cc, 8).to(DEV)
    z = torch.randn(N, 8, device=DEV)
    y = torch.randn(N, Cc, H, W, device=DEV).contiguous(memory_format=torch.channels_last)
    lo = torch.randn(N, Cc, H // 2, W // 2 + 2, device=DEV).contiguous(memory_format=torch.channels_last)
    res = []
    for half in (True, False):
        yy, ll = y.clone().requires_grad_(True), lo.clone().requires_grad_(True)
        skip = ll if half else F.interpolate(ll[..., 1:-1], scale_factor=2, mode="nearest").contiguous(memory_format=torch.channels_last)
        out = cbn_act_pad(yy, cbn, z, skip_nchw=skip, skip_off=1 if half else 0, skip_half=half, up=1, pad=2,
                          post_leaky=post_leaky, pad_mode=mode)
        g = torch.randn(out.shape, device=DEV, generator=torch.Generator(DEV).manual_seed(9))
        out.backward(g)
        res.append((out.detach(), yy.grad, ll.grad))
    for a, b, what in zip(res[0], res[1], ("output", "y gradient", "skip gradient")):
        assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max()), what


@pytest.mark.parametrize("symmetric", [True, False])
def test_fused_generator_matches_module_path(symmetric):
    from models import gan
    args = GC.make_args(128, 2)
    torch.manual_seed(123)
    G = gan.Generator(args, 64, symmetric=symmetric, mesh_head=True)
    with torch.no_grad():       # the mesh head is zero-initialised: give it a signal
        G.conv_mesh.weight.normal_(0, 0.02)
    G = G.to(DEV).train()
    import copy
    U = copy.deepcopy(G)
    U.disable_fusion = True
    z, c = [t.to(DEV) for t in GC.inputs(args, B=4)[:2]]
    outs = []
    for m in (G, U):
        a, b = m(z, c)
        (a.square().mean() + b.square().mean()).backward()
        outs.append(([a.detach(), b.detach()], {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None},
                     {n: b.clone() for n, b in m.named_buffers()}))
    (fa, ga, ba), (fb, gb, bb) = outs
    # test_bank_gpu.py's bounds for the bank against the module path: the bank feeds weights rounded to the nearest tf32
    # (here P, rounded once after the sum), the module path lets the tensor cores truncate them
    for a, b in zip(fa, fb):
        assert float((a - b).abs().max()) <= 1e-2 * float(b.abs().max())
    assert ga.keys() == gb.keys()
    floor = 2e-3 * max(float(g.norm()) for g in gb.values())
    bad = [(n, float(ga[n].norm()), float(gb[n].norm())) for n in gb
           if abs(float(ga[n].norm()) - float(gb[n].norm())) > 8e-2 * float(gb[n].norm()) + floor]
    assert not bad, bad[:10]
    for n in bb:
        if bb[n].is_floating_point():
            assert float((ba[n] - bb[n]).abs().max()) <= 1e-3 * float(bb[n].abs().max()) + 1e-5, n


@pytest.fixture
def up_recorder(monkeypatch):
    """Records the geometry of every call of the new helpers, and which layers reach the generic banked convolution."""
    import models.gan as gan
    rec = {"up": [], "generic_up2": []}
    for kind in ("fprop", "dgrad", "wgrad"):
        fn = getattr(C, "_up_" + kind)

        def wrapped(*args, _fn=fn, _kind=kind):
            rec["up"].append((_kind, tuple(a.shape if isinstance(a, torch.Tensor) else None for a in args)))
            return _fn(*args)
        monkeypatch.setattr(C, "_up_" + kind, wrapped)
    banked = gan.conv2d_banked

    def generic(x, lw, *args, **kw):
        if lw.wp is not None:                             # a layer the bank registered with up2
            rec["generic_up2"].append(tuple(x.shape))
        return banked(x, lw, *args, **kw)
    monkeypatch.setattr(gan, "conv2d_banked", generic)
    return rec


def _geom(kind, shapes):
    """(N, H, W, Cin, Cout, Csc) of one recorded call, from its tensors' shapes."""
    if kind == "fprop":                                   # xp, P, wsc, stats
        (N, H, Wp, Cin), (_, Cout, _), wsc = shapes[0], shapes[1], shapes[2]
        return N, H, Wp - 2, Cin, Cout, wsc[1] if wsc else 0
    if kind == "dgrad":                                   # gy, D4, gsc, Dsc
        (N, H2, W2, Cout), (_, Cin, _), gsc = shapes[0], shapes[1], shapes[2]
        return N, H2 // 2, W2 // 2, Cin, Cout, gsc[3] if gsc else 0
    (N, H2, W2, Cout), (_, H, Wp, Cin), gsc = shapes[0], shapes[1], shapes[3]   # gy, xp, df, gsc, dfsc
    return N, H, Wp - 2, Cin, Cout, gsc[3] if gsc else 0


def _check(rec, cfg, batches):
    table = {(n, H, W, Cin, Cout, Csc) for c, _, N, H, W, Cin, Cout, Csc in TABLE if c == cfg for n in batches}
    assert rec["up"], "no upsampled layer ran on the new helpers"
    for kind, shapes in rec["up"]:
        assert _geom(kind, shapes) in table, f"{cfg}: {kind} {shapes} is not in the per-layer table"
    assert {k for k, _ in rec["up"]} == {"fprop", "dgrad", "wgrad"}
    assert not rec["generic_up2"], f"{cfg}: an upsampled conv1 still runs on the generic path: {rec['generic_up2']}"


def _template(rings):
    import os
    import tempfile
    from oracle import mesh as M
    from rendering.mesh_template import MeshTemplate
    return MeshTemplate(M.write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), f"uvsphere_{rings}rings.obj"), rings=rings),
                        device=DEV)


def _steps(R, B, conditional, nd):
    from gan_training import GANTrainer
    args = types.SimpleNamespace(texture_resolution=R, conditional_class=conditional, conditional_color=False,
                                 conditional_text=False, norm_g='syncbatch', norm_d='none', n_classes=(200,), mask_output=True,
                                 texture_only=False, num_discriminators=nd, text_embedding_dim=256, latent_dim=64, loss='hinge',
                                 lr_g=1e-4, lr_d=4e-4, d_steps_per_g=2, mesh_regularization=1e-4, g_running_average_alpha=0.999,
                                 symmetric_g=True)
    torch.manual_seed(4321)
    tr = GANTrainer(args, mesh_template=_template(16), device=DEV)
    g = torch.Generator().manual_seed(77)
    alpha = (torch.rand(B, 1, R // 8, R // 8, generator=g) > 0.4).float()
    X_tex = (torch.rand(B, 3, R, R, generator=g) * 2 - 1).to(DEV)
    X_alpha = F.interpolate(alpha, size=(R, R), mode="bilinear", align_corners=False).to(DEV)
    X_mesh = (torch.randn(B, 3, 32, 32, generator=g) * 0.05).to(DEV)
    Cl = torch.randint(0, 200, (B, 1), generator=g).to(DEV)
    tr.g_step(X_alpha, Cl)
    tr.d_step(X_tex, X_alpha, X_mesh, Cl)
    torch.cuda.synchronize()


def test_cfg3_steps_use_the_up_helpers(up_recorder):
    _steps(256, 32, False, 2)
    _check(up_recorder, "cfg3", (32, 64))


def test_cfg5_steps_use_the_up_helpers(up_recorder):
    _steps(512, 8, True, 3)
    _check(up_recorder, "cfg5", (8, 16))
