"""Every convolution of the reconstruction workload (cfg4) and of the 512^2 GAN (cfg5) at its benchmark shape, against fp64.

cfg4: ReconstructionNetwork(symmetric=True, texture_res=128) at batch 50 and at 13 (one rank of four under DDP), on the
module path (b3d.conv.conv2d).  cfg5: the 512^2 generator at batch 8 and the three discriminators at 8 (generator step,
frozen) and 16 (discriminator step: fake and real images in one batch), through conv2d_banked with a WeightBank, as
MultiScaleDiscriminator calls it; their input gradients that carry the producer's LeakyReLU adjoint run with the mask and
the bias sums (b3d.conv.ActLink).

The dispatch of b3d_conv2d_tf32 / b3d_conv2d_wgrad_tf32 picks tile widths, row windows, strip launches, pixel tiles of
BW x BH x BI and K splits from N, H, W and the SM count, so these shapes reach launch geometries the cfg3 tables
(test_bench_shapes_gpu.py and friends) do not.  For each entry: forward and input gradient per image (images 0, N - 1 and
one of the last, partial image group of a tile when there is one), weight and bias gradients over the whole batch, each
within 4e-3 of the largest fp64 magnitude; the kernel instances every launch reports equal the ones tests/conv_plan.py
predicts.  test_tables_reach_the_geometries asserts from those plans that the tables reach the geometries they exist for,
and the two training-step tests record every convolution a real cfg4 / cfg5 iteration makes and find each in the tables."""
import collections
import inspect
import math

import pytest
import torch

import conv_plan as P

pytestmark = pytest.mark.gpu
TOL = 4e-3
DEV = "cuda:0"
SLOPE = 0.2


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# name, N, Cin, H, W (x-padded input), Cout, k, pad_y, stride, x_crop, bias, input gradient, masked input gradient,
# banked (conv2d_banked + WeightBank; else the module path), frozen (no weight gradient: the generator step's discriminators)
Entry = collections.namedtuple("Entry", "name N Cin H W Cout k pad_y stride x_crop bias dx masked banked frozen")


def _enc(name, Cin, H, W, Cout, k, pad_y, dx=True):
    return (name, Cin, H, W, Cout, k, pad_y, 2, 0, False, dx)


def _res(prefix, cin, mid, cout, H, W):
    """A residual block on an x-padded H x W input: conv1 cin -> mid, conv2 mid -> cout (3x3), 1x1 shortcut when cin != cout."""
    rows = [(prefix + ".conv1", cin, H, W, mid, 3, 1, 1, 0, False, True), (prefix + ".conv2", mid, H, W, cout, 3, 1, 1, 0, False, True)]
    if cin != cout:
        rows.append((prefix + ".short", cin, H, W, cout, 1, 0, 1, 1, False, True))
    return rows


# ReconstructionNetwork(symmetric=True, texture_res=128): encoder 256 -> 8 (stride 2), decoder on half-width maps
REC = ([_enc("conv1e", 4, 256, 260, 64, 5, 2, dx=False), _enc("conv2e", 64, 128, 130, 128, 3, 1),
        _enc("conv3e", 128, 64, 66, 256, 3, 1), _enc("conv4e", 256, 32, 34, 512, 3, 1), _enc("conv5e", 512, 16, 18, 64, 3, 1)]
       + _res("blk1", 256, 256, 512, 4, 4) + _res("blk2", 512, 512, 256, 8, 6) + _res("blk3", 256, 256, 256, 16, 10)
       + _res("blk3b_tex", 256, 256, 256, 32, 18) + _res("blk4_tex", 256, 256, 128, 64, 34)
       + _res("blk5_tex", 128, 128, 64, 128, 66) + _res("blk4_mesh", 256, 256, 64, 32, 18)
       + [("conv_tex", 64, 128, 68, 3, 5, 2, 1, 0, True, True), ("conv_mesh", 64, 32, 20, 3, 5, 2, 1, 0, True, True)])
CFG4 = [Entry(r[0], n, *r[1:], False, False, False) for n in (50, 13) for r in REC]

# 512^2 generator (half-width maps, ResBlockUp: conv1 cin -> min(cin, cout))
GEN = (_res("G.blk1", 512, 512, 512, 8, 6) + _res("G.blk2", 512, 256, 256, 16, 10) + _res("G.blk3a", 256, 256, 256, 32, 18)
       + _res("G.blk3b", 256, 256, 256, 64, 34) + _res("G.blk4", 256, 128, 128, 128, 66) + _res("G.blk5", 128, 128, 128, 256, 130)
       + _res("G.blk6", 128, 64, 64, 512, 258) + [("G.conv_final", 64, 512, 260, 3, 5, 2, 1, 0, True, True)]
       + _res("G.blk3_mesh", 256, 64, 64, 32, 18) + [("G.conv_mesh", 64, 32, 20, 3, 5, 2, 1, 0, True, True)])
# discriminators: d1 (512^2, stride-2 stem), d2 (the mesh discriminator at 32^2, 11 channels), d3 (downsample 4: 128^2,
# 5x5 stem folded from the raw 8-channel input); name, Cin, H, W, Cout, k, pad_y, stride, masked input gradient
DIS = [("d1.conv1", 8, 512, 514, 64, 4, 1, 2, False), ("d1.conv2", 64, 256, 258, 128, 4, 1, 2, True),
       ("d1.conv3", 128, 128, 130, 256, 4, 1, 2, True), ("d1.conv4", 256, 64, 66, 512, 4, 1, 2, True),
       ("d1.conv5", 512, 32, 36, 1, 5, 2, 1, False),
       ("d2.conv1", 11, 32, 36, 64, 5, 2, 1, False), ("d2.conv2", 64, 32, 34, 128, 4, 1, 2, True),
       ("d2.conv3", 128, 16, 18, 256, 4, 1, 2, True), ("d2.conv4", 256, 8, 12, 1, 5, 2, 1, False),
       ("d3.conv1", 8, 128, 132, 64, 5, 2, 1, False), ("d3.conv2", 64, 128, 130, 128, 4, 1, 2, True),
       ("d3.conv3", 128, 64, 66, 256, 4, 1, 2, True), ("d3.conv4", 256, 32, 34, 512, 4, 1, 2, True),
       ("d3.conv5", 512, 16, 20, 1, 5, 2, 1, False)]
CFG5 = ([Entry(r[0], 8, *r[1:], False, True, False) for r in GEN]
        + [Entry(n, N, ci, h, w, co, k, py, st, 0, True, N == 8 or not n.endswith("conv1"), m, True, N == 8)
           for N in (8, 16) for (n, ci, h, w, co, k, py, st, m) in DIS])
TABLE = CFG4 + CFG5


def _calls(e, sms):
    """The launch-helper calls of one entry (tests/conv_plan.py): the autograd pass, plus the masked input gradient."""
    calls = P.layer_calls(e.N, e.Cin, e.H, e.W, e.Cout, e.k, e.pad_y, e.stride, e.x_crop, e.dx and not e.masked, not e.frozen,
                          banked=e.banked, sms=sms)
    if e.masked:
        calls.append(P.Call("dgrad", e.N, e.H, e.W, P.r32(e.Cin), e.Cout, e.k, e.k, e.pad_y, e.stride, e.x_crop, masked=True))
    return calls


def _workload_calls(e, sms):
    """The calls the networks make for this layer (the masked input gradient is the autograd one there)."""
    return P.layer_calls(e.N, e.Cin, e.H, e.W, e.Cout, e.k, e.pad_y, e.stride, e.x_crop, e.dx, not e.frozen, e.masked, e.banked, sms)


# ----------------------------------------------------------------------------------------------------------------------
# recording the launch helpers
# ----------------------------------------------------------------------------------------------------------------------
def _as_call(kind, fn, args, kwargs):
    a = inspect.signature(fn).bind(*args, **kwargs)
    a.apply_defaults()
    v = a.arguments
    if kind == "fprop":
        x, wt = v["x"], v["wt"]
        return P.Call("fprop", *x.shape[:3], x.shape[3], wt.shape[1], v["kh"], v["kw"], v["pad_y"], v["stride"], v["x_crop"],
                      v["fold_kh"], v["fold_pad"])
    if kind == "dgrad":
        gy, (H, W) = v["gy"], v["in_hw"]
        return P.Call("dgrad", gy.shape[0], H, W, v["wd"].shape[1], gy.shape[3], v["kh"], v["kw"], v["pad_y"], v["stride"],
                      v["x_crop"], masked=v["mask"] is not None)
    gy, x = v["gy"], v["x"]
    return P.Call("wgrad", *x.shape[:3], x.shape[3], gy.shape[3], v["kh"], v["kw"], v["pad_y"], v["stride"], v["x_crop"],
                  v["fold_kh"])


@pytest.fixture
def recorder(monkeypatch):
    """Wraps b3d.conv._fprop / _dgrad / _wgrad: a list of (Call, the kernel instances that call launched)."""
    import b3d.conv as C
    rec = []
    monkeypatch.setattr(C, "VARIANT_LOG", [])
    for kind in ("fprop", "dgrad", "wgrad"):
        fn = getattr(C, "_" + kind)

        def wrapped(*args, _fn=fn, _kind=kind, **kwargs):
            call = _as_call(_kind, _fn, args, kwargs)
            n0 = len(C.VARIANT_LOG)
            out = _fn(*args, **kwargs)
            rec.append((call, list(C.VARIANT_LOG[n0:])))
            return out
        monkeypatch.setattr(C, "_" + kind, wrapped)
    return rec


def _check_plans(rec, sms, where):
    for call, ran in rec:
        want = call.instances(sms)
        assert ran == want, f"{where}: {call} launched {ran}, conv_plan predicts {want}"


# ----------------------------------------------------------------------------------------------------------------------
# one layer against fp64
# ----------------------------------------------------------------------------------------------------------------------
def _ref_images(e, sms, kind):
    """The first image of the last image group of every launch whose tiles hold BI > 1 images and N % BI != 0, 0 and N - 1."""
    imgs = {}
    for c in _calls(e, sms):
        if c.kind == kind:
            for l in c.launches(sms):
                if l.partial_group:
                    imgs.setdefault(e.N // l.BI * l.BI, f"first of the last group of {l.BI} ({l.instance}, columns {l.x0}-{l.x1})")
    imgs.setdefault(0, "first")
    imgs.setdefault(e.N - 1, "last")
    return imgs


def _per_image(e, what, got, ref, imgs):
    assert bool(torch.isfinite(got).all()), f"{e.name} N={e.N}: {what} is not finite"
    for i, why in imgs.items():
        err, mag = float((got[i].double() - ref[i]).abs().max()), float(ref[i].abs().max())
        assert err <= TOL * mag, f"{e.name} N={e.N}: {what} of image {i} ({why}): max|err| {err:.3e} > {TOL} x {mag:.3e}"


def _whole(e, what, got, ref):
    assert bool(torch.isfinite(got).all()), f"{e.name} N={e.N}: {what} is not finite"
    err, mag = float((got.double() - ref).abs().max()), float(ref.abs().max())
    assert err <= TOL * mag, f"{e.name} N={e.N}: {what} over the batch: max|err| {err:.3e} > {TOL} x {mag:.3e}"


@pytest.mark.parametrize("e", TABLE, ids=[f"{e.name}-N{e.N}" for e in TABLE])
def test_layer_against_fp64(e, recorder):
    import b3d.conv as C
    from b3d.bank import WeightBank
    from models.gan import TCConv2d
    sms = _sms()
    g = torch.Generator().manual_seed(sum(map(ord, e.name)) + e.N)
    conv = TCConv2d(e.Cin, e.Cout, e.k, stride=e.stride, padding=(e.pad_y, 0), bias=e.bias)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) / math.sqrt(e.Cin * e.k * e.k))
        if e.bias:
            conv.bias.copy_(torch.randn(e.Cout, generator=g))
    conv = conv.to(DEV).requires_grad_(not e.frozen)
    x = torch.randn(e.N, e.Cin, e.H, e.W, generator=g).to(DEV).contiguous(memory_format=torch.channels_last)
    x.requires_grad_(e.dx and not e.masked)
    if e.banked:
        fold = e.stride == 1 and e.k > 1 and e.Cin * e.k <= 64
        lw = WeightBank({"c": conv}, fold=("c",) if fold else (), round_tf32=False).forward(True)["c"]
        y = C.conv2d_banked(x, lw, pad_y=e.pad_y, stride=e.stride, x_crop=e.x_crop)
    else:
        y = conv(x, x_crop=e.x_crop)
    gy = torch.randn(y.shape[0], y.shape[2], y.shape[3], y.shape[1], generator=g).to(DEV)
    wrt = ([x] if x.requires_grad else []) + ([conv.weight] + ([conv.bias] if e.bias else []) if not e.frozen else [])
    grads = list(torch.autograd.grad(y, wrt, gy.permute(0, 3, 1, 2))) if wrt else []
    gx = grads.pop(0) if x.requires_grad else None
    dw, db = (grads + [None, None])[:2]
    sums = None
    if e.masked:
        # the consumer side of an ActLink: LeakyReLU'(the producer's activation) in the epilogue, bias sums when trained
        mask = torch.randn(e.N, e.H, e.W, e.Cin, generator=g).to(DEV)
        sums = None if e.frozen else torch.zeros(2 * e.Cin, device=DEV, dtype=torch.float64)
        gx = C._dgrad(gy, lw.wd, (e.H, e.W), e.k, e.k, e.pad_y, e.stride, mask=mask, slope=SLOPE, sums=sums).permute(0, 3, 1, 2)
    torch.cuda.synchronize()

    wd, xd = conv.weight.detach().double(), x.detach().double()
    bd = conv.bias.detach().double() if e.bias else None
    xc = xd[..., e.x_crop:e.W - e.x_crop] if e.x_crop else xd
    gyd = gy.permute(0, 3, 1, 2).double()
    imgs = _ref_images(e, sms, "fprop")
    idx = sorted(imgs)
    ref_y = torch.nn.functional.conv2d(xc[idx], wd, bd, stride=e.stride, padding=(e.pad_y, 0))
    _per_image(e, "forward", y.detach(), dict(zip(idx, ref_y)), imgs)
    if gx is not None:
        imgs = _ref_images(e, sms, "dgrad")
        idx = sorted(imgs)
        r = torch.nn.grad.conv2d_input((len(idx), e.Cin, e.H, e.W - 2 * e.x_crop), wd, gyd[idx], stride=e.stride,
                                       padding=(e.pad_y, 0))
        r = torch.nn.functional.pad(r, (e.x_crop, e.x_crop))
        if e.masked:
            r = r * torch.where(mask[idx].permute(0, 3, 1, 2) >= 0, 1.0, SLOPE).double()
        _per_image(e, "input gradient", gx.detach(), dict(zip(idx, r)), imgs)
        if sums is not None:
            gsum = gx.detach().double().sum(dim=(0, 2, 3))
            err = float((sums[:e.Cin] - gsum).abs().max())
            assert err <= 2e-6 * float(gx.detach().double().abs().sum(dim=(0, 2, 3)).max()), (e.name, "bias sums", err)
            assert float(sums[e.Cin:].abs().max()) == 0.0, (e.name, "sums only")
    if dw is not None:
        _whole(e, "weight gradient", dw, torch.nn.grad.conv2d_weight(xc, wd.shape, gyd, stride=e.stride, padding=(e.pad_y, 0)))
    if db is not None:
        _whole(e, "bias gradient", db, gyd.sum(dim=(0, 2, 3)))

    # launch plans: the calls and, launch for launch, the kernel instances
    assert collections.Counter(c for c, _ in recorder) == collections.Counter(_calls(e, sms)), \
        (e.name, [c for c, _ in recorder], _calls(e, sms))
    _check_plans(recorder, sms, f"{e.name} N={e.N}")


# ----------------------------------------------------------------------------------------------------------------------
# the tables reach what they are for
# ----------------------------------------------------------------------------------------------------------------------
def test_tables_reach_the_geometries():
    """From the plans of every table entry at this device's SM count: the launch geometries that no cfg3 table reaches."""
    sms = _sms()
    plans = [(e, c, c.launches(sms)) for e in TABLE for c in _calls(e, sms)]
    launches = [(e, c, l) for e, c, ls in plans for l in ls]
    found = {}

    def reach(item, ok):
        found.setdefault(item, False)
        found[item] = found[item] or bool(ok)

    for e, c, l in launches:
        # 1. a 25-tap stride-2 forward on the 64-wide tiles, its weight gradient with a ragged K split
        reach("1 fwd 25 taps stride 2", c.kind == "fprop" and l.taps == 25 and l.sy == 2 and l.BN == 64)
        reach("1 wgrad 25 taps ragged", c.kind == "wgrad" and l.taps == 25 and c.stride == 2 and l.kslices % l.splits)
        # 2. stride-2 input gradients in unmerged parity classes, 64- and 128-wide, and 1-column strips with a partial group
        for bn in (64, 128):
            reach(f"2 unmerged classes {bn}", c.kind == "dgrad" and c.stride == 2 and l.ncls == 1 and l.BN == bn)
        reach("2 strip BW=1 partial group", c.kind == "dgrad" and c.stride == 2 and l.strip and l.BW == 1 and l.partial_group)
        # 3. tiny maps with 16 images per tile and a partial group: forward, input gradient, x-cropped shortcut
        for kind in ("fprop", "dgrad"):
            reach(f"3 BI=16 partial {kind}", c.kind == kind and l.BI == 16 and l.partial_group)
        reach("3 BI=16 partial x_crop", c.x_crop and l.BI == 16 and l.partial_group)
        # 4. 3x3 row windows with more than one 128-pixel tile per row
        for kind in ("fprop", "dgrad"):
            reach(f"4 rowwin 3 two tiles per row {kind}", c.kind == kind and l.rowwin == 3 and l.x1 - l.x0 >= 256)
        # 5. the unfolded 512^2 stem: 8 -> 32 channels, 4x4 / stride 2
        reach("5 stem fwd", c.kind == "fprop" and c.Cin == 32 and c.kh == 4 and c.stride == 2 and l.BN == 64)
        reach("5 stem wgrad", c.kind == "wgrad" and c.Cin == 32 and c.kh == 4 and l.instance == "wgrad_wgmma<64,3,3,2>")
        # 6. grids with fewer work items than SMs
        reach("6 fewer items than SMs", c.kind in ("fprop", "dgrad") and l.items < sms)
        reach("K split ragged", c.kind == "wgrad" and l.splits and l.kslices % l.splits)
    # 6. tile widths that flip with the batch
    widths = collections.defaultdict(set)
    for e, c, ls in plans:
        if c.kind in ("fprop", "dgrad"):
            widths[(e.name, c.kind)].add((e.N, ls[0].BN))
    flips = [k for k, v in widths.items() if len({bn for _, bn in v}) > 1]
    found["6 tile width flips with the batch"] = bool(flips)
    missing = sorted(k for k, v in found.items() if not v)
    print("reached:", sorted(k for k, v in found.items() if v), "widths flip in", flips)
    assert not missing, f"no table entry reaches: {missing}"


# ----------------------------------------------------------------------------------------------------------------------
# the tables cover the real training steps
# ----------------------------------------------------------------------------------------------------------------------
def _assert_covered(rec, sms, where):
    known = {c for e in TABLE for c in _workload_calls(e, sms)}
    _check_plans(rec, sms, where)
    missing = sorted({c for c, _ in rec if c not in known}, key=repr)
    assert rec and not missing, f"{where}: convolutions no table entry describes: {missing}"


def _template(rings):
    import os
    import tempfile
    from oracle import mesh as M
    from rendering.mesh_template import MeshTemplate
    return MeshTemplate(M.write_uvsphere_obj(os.path.join(tempfile.mkdtemp(), f"uvsphere_{rings}rings.obj"), rings=rings),
                        device=DEV)


def test_cfg4_step_is_covered(recorder):
    """One ReconTrainer step (optimize_z0, texture 128, batch 50) on a 31-ring template."""
    from reconstruction_training import ReconTrainer, default_args
    B, H = 50, 256
    torch.manual_seed(4321)
    tr = ReconTrainer(default_args(optimize_z0=True), _template(31), dataset_size=4722, device=DEV)
    g = torch.Generator().manual_seed(13)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1, 1, H), indexing="ij")
    disk = ((yy * yy + xx * xx) < 0.45).float()
    x_real = torch.rand(B, 4, H, H, generator=g) * 2 - 1
    x_real[:, 3] = disk
    x_real[:, :3] *= disk
    pscale = 0.55 + 0.3 * torch.rand(B, 1, generator=g)
    ptrans = (torch.rand(B, 3, generator=g) - 0.5) * 0.3
    rot = torch.nn.functional.normalize(torch.randn(B, 4, generator=g), dim=-1)
    idx = torch.randint(0, 2 * 4722, (B,), generator=g)
    tr.step(*(t.to(DEV) for t in (x_real, pscale, ptrans, rot, idx)))
    torch.cuda.synchronize()
    _assert_covered(recorder, _sms(), "cfg4 step")


def test_cfg5_steps_are_covered(recorder):
    """One generator and one discriminator step of the 512^2 class-conditional GAN with three discriminators, batch 8."""
    import types
    from gan_training import GANTrainer
    B, R = 8, 512
    args = types.SimpleNamespace(texture_resolution=R, conditional_class=True, conditional_color=False, conditional_text=False,
                                 norm_g='syncbatch', norm_d='none', n_classes=(200,), mask_output=True, texture_only=False,
                                 num_discriminators=3, text_embedding_dim=256, latent_dim=64, loss='hinge', lr_g=1e-4,
                                 lr_d=4e-4, d_steps_per_g=2, mesh_regularization=1e-4, g_running_average_alpha=0.999,
                                 symmetric_g=True)
    torch.manual_seed(4321)
    tr = GANTrainer(args, mesh_template=_template(16), device=DEV)
    g = torch.Generator().manual_seed(77)
    alpha = (torch.rand(B, 1, R // 8, R // 8, generator=g) > 0.4).float()
    X_tex = (torch.rand(B, 3, R, R, generator=g) * 2 - 1).to(DEV)
    X_alpha = torch.nn.functional.interpolate(alpha, size=(R, R), mode="bilinear", align_corners=False).to(DEV)
    X_mesh = (torch.randn(B, 3, 32, 32, generator=g) * 0.05).to(DEV)
    C = torch.randint(0, 200, (B, 1), generator=g).to(DEV)
    tr.g_step(X_alpha, C)
    tr.d_step(X_tex, X_alpha, X_mesh, C)
    torch.cuda.synchronize()
    _assert_covered(recorder, _sms(), "cfg5 steps")
