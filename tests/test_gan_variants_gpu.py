"""The GAN option variants on the fused CUDA path: norm_g instance / none, norm_d instance and the asymmetric (full-width,
circular) generator.

  * against tests/golden/gan_variants_reference.npz (the reference's modules on the CPU): one G step, one D step and an
    eval-mode generator forward per configuration, with test_gan_gpu.py's tolerances (activations 2e-2 of the largest
    magnitude, losses 2e-2, gradient norms 6e-2 + 2e-3 of the largest norm);
  * no torch fallback: F.instance_norm / batch_norm / interpolate / leaky_relu and torch's spectral-norm compute_weight
    raise during the fused G and D forward and backward;
  * the fused generator equals its module path (disable_fusion) within 1e-3 or twice the default configuration's gap;
  * the new glue (per-sample statistics, per-sample coupling terms, circular padding and its adjoint) against the same
    composition in fp64 torch at the discriminator's instance-norm layers of cfg3 (B 32 -> 64 in the D step) and at the
    generator's layer shapes down to blk1's 32-pixel samples: |kernel - fp64| <= 4 |torch fp32 - fp64| + 1e-6 max|fp64|;
  * edges: a near-constant channel, N = 1, eval == train, circular pad columns and the padding adjoint bit exact against
    b3d_pad_x_fwd / b3d_pad_x_bwd;
  * three GANTrainer steps, eager and replayed from captured CUDA graphs."""
import copy
import importlib
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import gan_common as GC                  # noqa: E402
import gan_variants_common as GV         # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
EPS = 1e-5


def close(a, ref, tol):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    err = float(np.abs(a - ref).max())
    lim = tol * max(float(np.abs(ref).max()), 1e-6)
    assert err <= lim, (err, lim)


def grad_norms_match(module, names, norms):
    params = dict(module.named_parameters())
    floor = 2e-3 * float(norms.max())
    for name, ref in zip(names, norms):
        got = float(params[str(name)].grad.norm())
        assert abs(got - ref) <= 6e-2 * ref + floor, (str(name), got, ref)


def build(name):
    from models import gan
    args, G, D = GV.build(gan, name)
    return args, G.to(DEV).train(), D.to(DEV).train()


# ------------------------------------------------------------------------------------------------ against the reference
@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "gan_variants_reference.npz"))


@pytest.mark.parametrize("name", list(GV.CONFIGS))
def test_steps_match_reference_golden(gold, name):
    from utils.losses import GANLoss
    k = name + "/"
    args, G, D = build(name)
    nd = args.num_discriminators
    crit = GANLoss('hinge', tensor=torch.cuda.FloatTensor)
    z, c, alpha, tex, mesh = [t.to(DEV) for t in GC.inputs(args, B=GV.B)]
    loss, pred_tex, pred_mesh, dout, mask = GC.g_step(G, D, crit, z, c, alpha)
    loss.mean().backward()
    close(pred_tex[:, :, ::16, ::16], gold[k + "tex_probe"], 2e-2)
    assert abs(float(pred_tex.double().sum()) - float(gold[k + "tex_sum"])) / pred_tex.numel() < 1e-3
    close(pred_mesh, gold[k + "mesh"], 2e-2)
    for i in range(nd):
        close(dout[i], gold[k + f"d_out{i}"], 2e-2)
    assert abs(float(loss) - float(gold[k + "g_loss"])) < 2e-2 * abs(float(gold[k + "g_loss"]))
    grad_norms_match(G, gold[k + "g_grad_names"], gold[k + "g_grad_norms"])
    G.zero_grad(); D.zero_grad()
    lf, lr, dout = GC.d_step(G, D, crit, z, c, alpha, tex, mesh)
    (lf.mean() + lr.mean()).backward()
    assert abs(float(lf) - float(gold[k + "d_loss_fake"])) < 2e-2 * abs(float(gold[k + "d_loss_fake"]))
    assert abs(float(lr) - float(gold[k + "d_loss_real"])) < 2e-2 * abs(float(gold[k + "d_loss_real"]))
    for i in range(nd):
        close(dout[i], gold[k + f"dd_out{i}"], 2e-2)
    grad_norms_match(D, gold[k + "d_grad_names"], gold[k + "d_grad_norms"])
    G.eval()
    with torch.no_grad():
        et, em = G(z, c)
    close(et[:, :, ::16, ::16], gold[k + "eval_tex_probe"], 2e-2)
    close(em, gold[k + "eval_mesh"], 2e-2)
    names, shapes, _ = GV.state_summary(G)
    assert names == [str(n) for n in gold[k + "g_state_names"]] and shapes == [str(s) for s in gold[k + "g_state_shapes"]]


# ------------------------------------------------------------------------------------------------ no torch fallback
def _raise(*a, **kw):
    raise AssertionError("torch fallback on the fused path")


@pytest.mark.parametrize("name", list(GV.CONFIGS))
def test_fused_path_uses_no_torch_fallback(name, monkeypatch):
    from utils.losses import GANLoss
    args, G, D = build(name)
    crit = GANLoss('hinge', tensor=torch.cuda.FloatTensor)
    z, c, alpha, tex, mesh = [t.to(DEV) for t in GC.inputs(args, B=GV.B)]
    with monkeypatch.context() as mp:
        for fn in ("instance_norm", "batch_norm", "interpolate", "leaky_relu"):
            mp.setattr(F, fn, _raise)
        mp.setattr(importlib.import_module("torch.nn.utils.spectral_norm").SpectralNorm, "compute_weight", _raise)
        loss = GC.g_step(G, D, crit, z, c, alpha)[0]
        loss.mean().backward()
        lf, lr, _ = GC.d_step(G, D, crit, z, c, alpha, tex, mesh)
        (lf.mean() + lr.mean()).backward()
    assert torch.isfinite(loss).all() and torch.isfinite(lf) and torch.isfinite(lr)


# ------------------------------------------------------------------------------------------------ fused == module path
def fused_gap(name):
    """Largest |fused - module path| / max|module path| of the generator's texture and mesh outputs, training and eval.
    Both sides take the convolutions' weights from the modules (torch's spectral-norm hook; the WeightBank rounds them
    to tf32 first, a separate 2^-11 difference), so what differs is the fused glue against the module path's norm,
    affine, LeakyReLU, add, upsample and padding."""
    if name == "default":
        from models import gan
        args = GC.make_args(256, 2)
        G = GC.build(gan, args)[0].to(DEV)
    else:
        args, G, _ = build(name)
    U = copy.deepcopy(G)
    G.disable_bank = True
    U.disable_fusion = True
    z, c = [t.to(DEV) for t in GC.inputs(args, B=GV.B)[:2]]
    errs = []
    for training in (True, False):
        G.train(training); U.train(training)
        a, b = G(z, c), U(z, c)
        for x, y in zip(a, b):
            errs.append((training, float((x - y).abs().max()) / float(y.abs().max())))
    print(name, errs)
    return max(e for _, e in errs)


@pytest.fixture(scope="module")
def default_gap():
    return fused_gap("default")


@pytest.mark.parametrize("name", list(GV.CONFIGS))
def test_fused_generator_equals_module_path(name, default_gap):
    """The glue's fp32 rounding differs from the module path's in the last bits; the tf32 convolutions that follow round
    their inputs to 2^-11, so single last-bit differences become tf32-rounding flips that accumulate over ~25 layers.  The
    default configuration (syncbatch, symmetric, the glue's batch-norm path) shows 2.5e-3 of the largest output on an
    H100 this way.  Each variant must stay within 1e-3 or twice the default configuration's gap."""
    gap = fused_gap(name)
    assert gap <= max(1e-3, 2 * default_gap), (name, gap, default_gap)


# ------------------------------------------------------------------------------------------------ glue against fp64
def _pad(h, pad, circular):
    if not pad:
        return h
    if circular:
        return torch.cat((h[..., -pad:], h, h[..., :pad]), dim=3)
    return F.pad(h, (pad, pad, 0, 0), mode='replicate')


def ref_glue(y, g, b, kind, skip=None, off=0, up=1, pad=1, post=False, circular=True, slope=0.2):
    """y [N,C,H,W]; g, b: gamma / beta rows [N or 1, C] (the affine is y_hat * (1 + g) + b) -> (out, pre)."""
    W = y.shape[3]
    if kind == 'instance':
        m = y.mean(dim=(2, 3), keepdim=True)
        v = y.var(dim=(2, 3), unbiased=False, keepdim=True)
        xh = (y - m) * (v + EPS).rsqrt()
    else:
        xh = y
    pre = xh * (1 + g[:, :, None, None]) + b[:, :, None, None]
    h = F.leaky_relu(pre, slope)
    if skip is not None:
        h = h + skip[..., off:off + W]
    if post:
        h = F.leaky_relu(h, slope)
    if up == 2:
        h = F.interpolate(h, scale_factor=2, mode='nearest')
    return _pad(h, pad, circular), pre


def _clear_kinks(y, g, b, kind, skip, off, post, thr=1e-4):
    """Move the rare elements whose activation inputs lie within thr of a kink 4 thr away from it (there fp32 and fp64 may
    take different branches: a difference of definition, not of accuracy)."""
    _, pre = ref_glue(y, g, b, kind, pad=0)
    a = (1 + g[:, :, None, None]) * ((y.var(dim=(2, 3), unbiased=False, keepdim=True) + EPS).rsqrt() if kind == 'instance' else 1)
    sgn = torch.where(pre >= 0, 1.0, -1.0).double()
    y = y + torch.where(pre.abs() < thr, sgn * 4 * thr / a, torch.zeros_like(pre))
    if skip is not None and post:
        W = y.shape[3]
        mid = F.leaky_relu(ref_glue(y, g, b, kind, pad=0)[1], 0.2) + skip[..., off:off + W]
        skip = skip.clone()
        skip[..., off:off + W] += torch.where(mid.abs() < thr, torch.where(mid >= 0, 1.0, -1.0).double() * 4 * thr,
                                              torch.zeros_like(mid))
    return y, skip


def run_glue(N, C, H, W, kind, cbn=True, up=1, pad=1, skip=None, post=False, circular=True, seed=0, const_channel=False,
             training=True):
    """kind 'instance' / 'none'.  cbn: a generator ConditionalBatchNorm2d (per-sample gamma / beta rows of a CBNBatch);
    else a discriminator InstanceNorm2d(affine=True) through in_act_pad.  skip: None, 'id' (offset 1) or 'sc' (offset 0).
    -> (kernel output, the fp64 reference output)."""
    from b3d.ew import CBNBatch, CIRCULAR, REPLICATE, cbn_act_pad, in_act_pad
    from models.gan import ConditionalBatchNorm2d
    gen = torch.Generator().manual_seed(2000 + seed)
    rn = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64).to(DEV)
    off = 1 if skip == 'id' else 0
    mu, sd = 0.5 * rn(C), 0.5 + 1.5 * torch.rand(C, generator=gen, dtype=torch.float64).to(DEV)
    y = rn(N, C, H, W) * sd[None, :, None, None] + mu[None, :, None, None]
    if const_channel:                           # per-sample variance ~ eps / 100: the eps under the root dominates
        y[:, 1] = (EPS / 100) ** 0.5 * rn(N, H, W)
    sk = rn(N, C, H, W + (2 if skip == 'id' else 0)) if skip else None
    if cbn:
        gb = 0.3 * rn(N, 2 * C)
        g, b = gb[:, :C], gb[:, C:]
    else:
        w, bias = 0.6 + 0.8 * torch.rand(C, generator=gen, dtype=torch.float64).to(DEV), 0.2 * rn(C)
        g, b = (w - 1)[None], bias[None]
    y, sk = _clear_kinks(y, g, b, kind, sk, off, post)
    y = y.float().double()
    sk = sk.float().double() if sk is not None else None
    wout = rn(N, C, up * H, up * W + 2 * pad)

    leaf = lambda t, dt: t.detach().to(dt, copy=True).requires_grad_(True)
    ref = {}
    for dt in (torch.float64, torch.float32):
        yy = leaf(y, dt)
        ss = leaf(sk, dt) if sk is not None else None
        if cbn:
            gg = leaf(gb, dt)
            out, _ = ref_glue(yy, gg[:, :C], gg[:, C:], kind, ss, off, up, pad, post, circular)
        else:
            ww, bb = leaf(w, dt), leaf(bias, dt)
            out, _ = ref_glue(yy, (ww - 1)[None], bb[None], kind, ss, off, up, pad, post, circular)
        (out * wout.to(dt)).sum().backward()
        ref[dt] = dict(out=out, gy=yy.grad, gs=ss.grad if ss is not None else None,
                       gp=[gg.grad] if cbn else [ww.grad, bb.grad])

    yk = y.detach().float().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    skk = sk.detach().float().contiguous(memory_format=torch.channels_last).requires_grad_(True) if sk is not None else None
    pm = CIRCULAR if circular else REPLICATE
    if cbn:
        m = ConditionalBatchNorm2d(types.SimpleNamespace(norm_g=kind), C, 16).to(DEV).train(training)
        cb = CBNBatch([m], torch.zeros(N, 16, device=DEV))
        cb.gb = gb.detach().float().requires_grad_(True)
        out = cbn_act_pad(yk, m, None, skip_nchw=skk, skip_off=off, up=up, pad=pad, post_leaky=post, cb=cb, pad_mode=pm)
        params = [cb.gb]
    else:
        norm = torch.nn.InstanceNorm2d(C, affine=True).to(DEV).train(training)
        with torch.no_grad():
            norm.weight.copy_(w.float()); norm.bias.copy_(bias.float())
        out = in_act_pad(yk, norm, pad, pm)
        params = [norm.weight, norm.bias]
    (out * wout.float()).sum().backward()
    from cbn_common import assert_close
    tag = f"{kind} {'cbn' if cbn else 'in'} N{N} C{C} {H}x{W} up{up} pad{pad} {'circ' if circular else 'repl'}"
    assert_close(tag + " out", out, ref[torch.float64]["out"], ref[torch.float32]["out"], 1e-4)
    assert_close(tag + " dy", yk.grad, ref[torch.float64]["gy"], ref[torch.float32]["gy"], 1e-3)
    if skk is not None:
        assert_close(tag + " dskip", skk.grad, ref[torch.float64]["gs"], ref[torch.float32]["gs"], 1e-3)
    for p, r64, r32 in zip(params, ref[torch.float64]["gp"], ref[torch.float32]["gp"]):
        assert_close(tag + " d(gamma, beta)", p.grad, r64, r32, 1e-3)
    return out.detach(), ref[torch.float64]["out"]


# the discriminators' instance-norm layers in cfg3's D step (B 32 fake + 32 real): d1 conv2..conv4, d2 conv2..conv3
D_LAYERS = [(128, 128, 128, 1), (256, 64, 64, 1), (512, 32, 32, 2), (128, 16, 16, 1), (256, 8, 8, 2)]


@pytest.mark.parametrize("C,H,W,pad", D_LAYERS)
def test_discriminator_instance_glue_against_fp64(C, H, W, pad):
    run_glue(64, C, H, W, 'instance', cbn=False, pad=pad, seed=C + H)


# generator layers (C, H, W of the conv output, up, pad, skip, post): blk1 at 32 pixels per sample (symmetric 8 x 4) and
# 64 (asymmetric 8 x 8), blk2's shortcut, blk6's post-activation into the 5x5 head's pad 2
G_LAYERS = [(512, 8, 4, 1, 1, None, False), (512, 8, 4, 2, 1, 'id', False), (512, 8, 8, 2, 1, 'id', False),
            (256, 16, 8, 2, 1, 'sc', False), (64, 128, 64, 1, 2, 'sc', True), (64, 32, 32, 1, 2, 'sc', True)]


@pytest.mark.parametrize("kind", ["instance", "none"])
@pytest.mark.parametrize("circular", [False, True])
@pytest.mark.parametrize("C,H,W,up,pad,skip,post", G_LAYERS)
def test_generator_glue_against_fp64(kind, circular, C, H, W, up, pad, skip, post):
    run_glue(32, C, H, W, kind, cbn=True, up=up, pad=pad, skip=skip, post=post, circular=circular, seed=C + W)


# ------------------------------------------------------------------------------------------------ edges
def test_near_constant_channel():
    run_glue(8, 64, 16, 8, 'instance', cbn=True, up=2, pad=1, skip='id', const_channel=True)
    run_glue(8, 128, 16, 16, 'instance', cbn=False, pad=1, const_channel=True)


@pytest.mark.parametrize("kind", ["instance", "none"])
def test_single_sample(kind):
    run_glue(1, 512, 8, 4, kind, cbn=True, up=2, pad=1, skip='id', circular=False)
    run_glue(1, 256, 16, 16, kind, cbn=True, up=2, pad=1, skip='sc')
    if kind == 'instance':
        run_glue(1, 256, 8, 8, 'instance', cbn=False, pad=2)


def test_instance_norm_eval_equals_train():
    a, _ = run_glue(4, 128, 16, 8, 'instance', cbn=True, up=2, pad=1, skip='id', training=True)
    b, _ = run_glue(4, 128, 16, 8, 'instance', cbn=True, up=2, pad=1, skip='id', training=False)
    assert torch.equal(a, b)
    a, _ = run_glue(4, 256, 8, 8, 'instance', cbn=False, pad=2, training=True)
    b, _ = run_glue(4, 256, 8, 8, 'instance', cbn=False, pad=2, training=False)
    assert torch.equal(a, b)


@pytest.mark.parametrize("up,pad,W", [(1, 1, 8), (1, 2, 4), (2, 1, 4), (2, 2, 8), (1, 4, 4)])
def test_circular_pad_columns_bit_exact(up, pad, W):
    from b3d.ew import CIRCULAR, pad_x
    out, _ = run_glue(2, 64, 8, W, 'instance', cbn=True, up=up, pad=pad, skip='id')
    assert torch.equal(out, pad_x(out[..., pad:out.shape[3] - pad].contiguous(memory_format=torch.channels_last), pad, CIRCULAR))


@pytest.mark.parametrize("pad,W", [(1, 8), (2, 4), (2, 2), (3, 5)])
def test_padding_adjoint_bit_exact(pad, W):
    """No normalisation, gamma = beta = 0 and slope 1: the backward is exactly the padding's adjoint."""
    from b3d.ew import CBNBatch, CIRCULAR, _CBNActPad, identity_norm, pad_x
    from models.gan import ConditionalBatchNorm2d
    N, C, H = 3, 32, 6
    m = ConditionalBatchNorm2d(types.SimpleNamespace(norm_g='none'), C, 16).to(DEV)
    assert m.norm is identity_norm
    cb = CBNBatch([m], torch.zeros(N, 16, device=DEV))
    cb.gb = torch.zeros(N, 2 * C, device=DEV)
    y = torch.randn(N, H, W, C, device=DEV).requires_grad_(True)
    g = torch.randn(N, H, W + 2 * pad, C, device=DEV)
    out = _CBNActPad.apply(y, cb.gb, cb, id(m), m.norm, None, 0, 1, pad, False, None, 1.0, CIRCULAR)
    out.backward(g)
    x = y.detach().permute(0, 3, 1, 2).requires_grad_(True)
    ref = pad_x(x, pad, CIRCULAR)
    assert torch.equal(out.permute(0, 3, 1, 2), ref)
    ref.backward(g.permute(0, 3, 1, 2))
    assert torch.equal(y.grad, x.grad.permute(0, 2, 3, 1))


# ------------------------------------------------------------------------------------------------ training + graph capture
def _trainer(name, seed):
    import bench
    from gan_training import GANTrainer
    args = bench.gan_args(256, 2)
    cfg = GV.CONFIGS[name]
    args.norm_g, args.norm_d, args.symmetric_g = cfg["norm_g"], cfg["norm_d"], cfg["symmetric"]
    torch.manual_seed(seed)
    return GANTrainer(args, mesh_template=None, device=DEV, capturable=True)


def _batches(n, seed, B=2):
    args = GC.make_args(256, 2)
    out = []
    for i in range(n):
        z, c, alpha, tex, mesh = GC.inputs(args, B=B, seed=seed + i)
        out.append(dict(X_tex=tex.to(DEV), X_alpha=alpha.to(DEV), X_mesh=mesh.to(DEV), C=c.to(DEV), noise=z.to(DEV)))
    return out


@pytest.mark.parametrize("name", ["cfg1", "cfg3"])
def test_trainer_steps_eager_and_graph_replay(name):
    """Three steps (G, D, D) after a warm-up G and D step: eager versus replays of captured G / D step graphs."""
    warm, batches = _batches(2, 50), _batches(3, 60)
    eager, again, cap = _trainer(name, 7), _trainer(name, 7), _trainer(name, 7)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                   # the Adams' capturable state is created outside the capture
        for tr in (eager, again, cap):
            tr.g_step(warm[0]["X_alpha"], warm[0]["C"], warm[0]["noise"])
            tr.d_step(warm[1]["X_tex"], warm[1]["X_alpha"], warm[1]["X_mesh"], warm[1]["C"], warm[1]["noise"])
    torch.cuda.current_stream().wait_stream(side)
    static = {k: v.clone() for k, v in batches[0].items()}
    gg, gd = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(gg):
        lg = cap.g_step(static["X_alpha"], static["C"], static["noise"])
    with torch.cuda.graph(gd):
        ld = cap.d_step(static["X_tex"], static["X_alpha"], static["X_mesh"], static["C"], static["noise"])
    losses = []
    for i, b in enumerate(batches):
        is_g = i == 0
        le = [tr.g_step(b["X_alpha"], b["C"], b["noise"]) if is_g else
              tr.d_step(b["X_tex"], b["X_alpha"], b["X_mesh"], b["C"], b["noise"]) for tr in (eager, again)]
        for k, v in b.items():
            static[k].copy_(v)
        (gg if is_g else gd).replay()
        losses.append([float(v) for v in le] + [float(lg if is_g else ld)])
    # the weight-gradient split-K atomics round differently from run to run (and Adam's first steps turn a gradient that
    # cancels to ~0 into a full +-lr step either way): the replayed graphs must stay within 4x the spread of two eager runs
    spread = max(abs(a - b) for a, b, _ in losses)
    print(name, "losses (eager, eager again, graph)", losses)
    for a, _, c in losses:
        assert abs(c - a) <= 4 * spread + 1e-5 * abs(a), losses
    pe, pa = dict(eager.trainer.named_parameters()), dict(again.trainer.named_parameters())
    d_again = max(float((pa[n] - p).abs().max()) for n, p in pe.items())
    d_cap = 0.0
    for n, p in cap.trainer.named_parameters():
        assert torch.isfinite(p).all(), n
        d_cap = max(d_cap, float((p - pe[n]).abs().max()))
    print(name, "largest parameter difference: eager again", d_again, "graph", d_cap)
    assert d_cap <= 4 * d_again + 1e-6, (d_cap, d_again)
