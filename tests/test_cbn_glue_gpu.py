"""The fused batch-norm glue of csrc/ew_kernels.cu (b3d_bn_sums, b3d_cbn_prepare, b3d_cbn_act_fwd, b3d_cbn_act_bwd1,
b3d_cbn_bwd_reduce, b3d_cbn_act_bwd2 through b3d.ew.cbn_act_pad / bn_act_pad) against the same composition in plain fp64
torch (tests/cbn_common.py), layer by layer, at every shape the generator and the reconstruction decoder use and at the
kernels' edges.

Tolerance: |kernel - fp64| <= 4 |torch fp32 - fp64| + 1e-6 max|fp64| (the error fp32 arithmetic alone makes on the same
composition), capped at 1e-4 of the largest magnitude for outputs and 1e-3 for gradients.  Pad columns, the four children
of an upsampled pixel and the untouched pad columns of a pitched skip gradient are checked bit for bit."""
import copy
import ctypes
import types

import pytest
import torch
import torch.nn.functional as F

from cbn_common import EMB, EPS, assert_close, clear_kinks, make_bn, make_cbn, ref_glue

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
OUT_CEIL, GRAD_CEIL = 1e-4, 1e-3


def L(C, H, W, up=1, pad=1, skip=None, post=False, slope=0.2):
    """One fused call: y [N,C,H,W] -> [N,C,up*H,up*W + 2*pad]; skip None, 'id' (the block's padded input, read at
    pixel offset 1) or 'sc' (a 1x1-shortcut output, offset 0)."""
    return types.SimpleNamespace(C=C, H=H, W=W, up=up, pad=pad, skip=skip, post=post, slope=slope,
                                 off=1 if skip == 'id' else 0)


def _randn(gen, *shape):
    return torch.randn(*shape, generator=gen, dtype=torch.float64)


def _structure(out, up, pad, W):
    """Bit-exact structure of a fused output: replicate-pad columns, identical x2 children."""
    if pad:
        assert torch.equal(out[..., :pad], out[..., pad:pad + 1].expand_as(out[..., :pad])), "left pad columns"
        assert torch.equal(out[..., -pad:], out[..., -pad - 1:-pad].expand_as(out[..., -pad:])), "right pad columns"
    if up == 2:
        inner = out[..., pad:pad + 2 * W]
        a = inner[:, :, 0::2, 0::2]
        for t in (inner[:, :, 1::2, 0::2], inner[:, :, 0::2, 1::2], inner[:, :, 1::2, 1::2]):
            assert torch.equal(a, t), "x2 children differ"


def run_glue(N, layers, kind='cbn', chain=False, seed=0, training=True, channels_last=True, bn_kw=None, const_channel=False):
    """Kernel path and fp64 / fp32 torch paths of the same layers; checks outputs, every gradient and the running buffers.
    kind 'cbn': ConditionalBatchNorm2d layers sharing one CBNBatch (gamma / beta GEMM and gradient sink) as in the
    generator; 'bn': BatchNorm2d layers through bn_act_pad (BNAffine) as in the reconstruction decoder.  chain: layer i's
    input is its own tensor + 0.25 x the interior of layer i-1's output (its first C_i channels), so the layers' backward passes run last to first."""
    from b3d.ew import CBNBatch, bn_act_pad, cbn_act_pad
    bn_kw = bn_kw or {}
    gen = torch.Generator().manual_seed(1000 + seed)
    mods = [(make_cbn if kind == 'cbn' else make_bn)(l.C, seed + i, **bn_kw).to(DEV).train(training) for i, l in enumerate(layers)]
    norms = [m.norm if kind == 'cbn' else m for m in mods]
    state0 = [(n.running_mean.clone(), n.running_var.clone(), int(n.num_batches_tracked)) if n.running_mean is not None else None
              for n in norms]
    batch_stats = [training or n.running_mean is None for n in norms]
    runs = [None if bs else (n.running_mean, n.running_var) for bs, n in zip(batch_stats, norms)]
    params = [[p.detach().double() for p in ((m.fc_gamma.weight, m.fc_gamma.bias, m.fc_beta.weight, m.fc_beta.bias)
                                            if kind == 'cbn' else (m.weight, m.bias))] for m in mods]
    z = _randn(gen, N, EMB).float().double().to(DEV)

    def rows(P, zz):
        if kind == 'cbn':
            return F.linear(zz, P[0], P[1]), F.linear(zz, P[2], P[3])
        return (P[0] - 1)[None], P[1][None]

    ys, skips, wouts = [], [], []
    for i, l in enumerate(layers):
        mu = 0.5 * _randn(gen, l.C)
        sd = 0.5 + 1.5 * torch.rand(l.C, generator=gen, dtype=torch.float64)
        y = _randn(gen, N, l.C, l.H, l.W) * sd[None, :, None, None] + mu[None, :, None, None]
        if const_channel and i == 0:                    # batch variance ~ eps / 4: +eps and clamp(eps) differ by 10 %
            y[:, 1] = (EPS / 4) ** 0.5 * _randn(gen, N, l.H, l.W)
        ys.append(y.to(DEV))
        skips.append(None if l.skip is None else _randn(gen, N, l.C, l.H, l.W + (2 if l.skip == 'id' else 0)).to(DEV))
        wouts.append(_randn(gen, N, l.C, l.up * l.H, l.up * l.W + 2 * l.pad).to(DEV))

    def feed(y, prev, l):                              # chained: + 0.25 x the previous output's interior
        return y + 0.25 * prev[:, :l.C, :, 1:-1] if chain and prev is not None else y

    def compose(ys_, skips_, P_, zz):
        outs, stats, prev = [], [], None
        for i, l in enumerate(layers):
            y = feed(ys_[i], prev, l)
            g, b = rows(P_[i], zz)
            out, _, _, m, v = ref_glue(y, g, b, skips_[i], l.off, l.up, l.pad, l.post, l.slope, runs[i])
            outs.append(out)
            stats.append((m, v))
            prev = out
        return outs, stats

    # move the rare pixels that sit on an activation kink off it (cbn_common.clear_kinks), layer by layer
    with torch.no_grad():
        prev = None
        for i, l in enumerate(layers):
            y = feed(ys[i], prev, l)
            g, b = rows(params[i], z)
            dy, dsk = clear_kinks(y, g, b, skips[i], l.off, l.post, l.slope, runs[i])
            ys[i] = (ys[i] + dy).float().double()
            if dsk is not None:
                skips[i] = skips[i] + dsk
            if skips[i] is not None:
                skips[i] = skips[i].float().double()
            prev = ref_glue(feed(ys[i], prev, l), g, b, skips[i], l.off, l.up, l.pad,
                            l.post, l.slope, runs[i])[0]

    ref = {}
    for dt in (torch.float64, torch.float32):
        ys_ = [y.to(dt, copy=True).requires_grad_(True) for y in ys]
        sk_ = [s.to(dt, copy=True).requires_grad_(True) if s is not None else None for s in skips]
        P_ = [[p.to(dt, copy=True).requires_grad_(True) for p in P] for P in params]
        zz = z.to(dt, copy=True).requires_grad_(True)
        outs, stats = compose(ys_, sk_, P_, zz)
        sum((o * w.to(dt)).sum() for o, w in zip(outs, wouts)).backward()
        ref[dt] = dict(outs=outs, stats=stats, gy=[y.grad for y in ys_], gs=[s.grad if s is not None else None for s in sk_],
                       gp=[[p.grad for p in P] for P in P_], gz=zz.grad)

    fmt = torch.channels_last if channels_last else torch.contiguous_format
    yk = [y.detach().float().contiguous(memory_format=fmt).requires_grad_(True) for y in ys]
    sk = [s.detach().float().contiguous(memory_format=fmt).requires_grad_(True) if s is not None else None for s in skips]
    zk = z.detach().float().requires_grad_(True)
    cb = CBNBatch(mods, zk) if kind == 'cbn' else None
    outs, prev = [], None
    for i, l in enumerate(layers):
        y = feed(yk[i], prev, l)
        if kind == 'cbn':
            assert l.slope == 0.2
            o = cbn_act_pad(y, mods[i], zk, skip_nchw=sk[i], skip_off=l.off, up=l.up, pad=l.pad, post_leaky=l.post, cb=cb)
        else:
            o = bn_act_pad(y, mods[i], skip_nchw=sk[i], skip_off=l.off, up=l.up, pad=l.pad, post_relu=l.post, slope=l.slope)
        outs.append(o)
        prev = o
    sum((o * w.float()).sum() for o, w in zip(outs, wouts)).backward()
    torch.cuda.synchronize()

    r64, r32 = ref[torch.float64], ref[torch.float32]
    pnames = ("fc_gamma.weight", "fc_gamma.bias", "fc_beta.weight", "fc_beta.bias") if kind == 'cbn' else ("weight", "bias")
    for i, l in enumerate(layers):
        assert_close(f"out[{i}]", outs[i], r64["outs"][i], r32["outs"][i], OUT_CEIL)
        _structure(outs[i].detach(), l.up, l.pad, l.W)
        assert_close(f"d y[{i}]", yk[i].grad, r64["gy"][i], r32["gy"][i], GRAD_CEIL)
        if sk[i] is not None:
            assert_close(f"d skip[{i}]", sk[i].grad, r64["gs"][i], r32["gs"][i], GRAD_CEIL)
            if l.off:                                       # pitched gskip: the pad columns get no gradient at all
                assert torch.all(sk[i].grad[..., :l.off] == 0) and torch.all(sk[i].grad[..., l.off + l.W:] == 0)
        for j, name in enumerate(pnames):
            p = (mods[i].fc_gamma.weight, mods[i].fc_gamma.bias, mods[i].fc_beta.weight, mods[i].fc_beta.bias)[j] \
                if kind == 'cbn' else (mods[i].weight, mods[i].bias)[j]
            assert_close(f"d {name}[{i}]", p.grad, r64["gp"][i][j], r32["gp"][i][j], GRAD_CEIL)
        # running buffers: momentum update with the unbiased batch variance (F.batch_norm), or untouched
        n, s0 = norms[i], state0[i]
        if s0 is None:
            continue
        if training and n.track_running_stats:
            m64, v64 = r64["stats"][i]
            cnt = N * l.H * l.W
            f = n.momentum if n.momentum is not None else 1.0 / (s0[2] + 1)
            rm_ref = (1 - f) * s0[0].double() + f * m64
            rv_ref = (1 - f) * s0[1].double() + f * v64 * cnt / max(cnt - 1, 1)
            assert float((n.running_mean.double() - rm_ref).abs().max()) <= 2e-6 * max(1.0, float(rm_ref.abs().max()))
            assert float((n.running_var.double() - rv_ref).abs().max()) <= 2e-6 * max(1.0, float(rv_ref.abs().max()))
            assert int(n.num_batches_tracked) == s0[2] + 1
        else:
            assert torch.equal(n.running_mean, s0[0]) and torch.equal(n.running_var, s0[1])
            assert int(n.num_batches_tracked) == s0[2]
    if kind == 'cbn':
        assert_close("d z", zk.grad, r64["gz"], r32["gz"], GRAD_CEIL)


# ---------------------------------------------------------------------------------------------------------------------
# every fused call of the networks at its real shape
# ---------------------------------------------------------------------------------------------------------------------
# generator at 256^2 (cfg3, batch 32) + blk3b of the 512^2 architecture: name, C_in, C_out, map H x W at the block's
# input, upsample, pad of the consumer, LeakyReLU after the residual add
GEN_BLOCKS = [("blk1", 512, 512, 8, 4, 2, 1, False), ("blk2", 512, 256, 16, 8, 2, 1, False),
              ("blk3a", 256, 256, 32, 16, 2, 1, False), ("blk3b", 256, 256, 64, 32, 2, 1, False),
              ("blk4", 256, 128, 64, 32, 2, 1, False), ("blk5", 128, 128, 128, 64, 2, 1, False),
              ("blk6", 128, 64, 256, 128, 1, 2, True), ("blk3_mesh", 256, 64, 32, 16, 1, 2, True)]


@pytest.mark.parametrize("blk", GEN_BLOCKS, ids=[b[0] for b in GEN_BLOCKS])
def test_generator_block_glue(blk):
    """ResBlockUp.forward_fused's two calls: norm1 (-> pad 1 for conv2) and norm2 (+ identity skip read from the padded
    input at offset 1, or + the 1x1 shortcut; -> x2 upsample + pad 1, or pad 2 + LeakyReLU for blk6 / blk3_mesh), one
    CBNBatch for both: the gradients of fc_gamma / fc_beta / z come out of the shared sink that norm1 closes."""
    name, cin, cout, H, W, up, pad, post = blk
    skip = 'id' if cin == cout else 'sc'
    print(name)
    run_glue(32, [L(cout, H, W), L(cout, H, W, up, pad, skip, post)], kind='cbn', chain=True, seed=len(name))


# reconstruction decoder as the benchmark trains it (texture_res 128, symmetric: half-width maps): name, C_in, C_out, H x W
# at the block's input, up, pad, ReLU after add
REC_BLOCKS = [("blk1", 256, 512, 4, 2, 2, 1, False), ("blk2", 512, 256, 8, 4, 2, 1, False), ("blk3", 256, 256, 16, 8, 2, 1, False),
              ("blk3b_tex", 256, 256, 32, 16, 2, 1, False), ("blk4_tex", 256, 128, 64, 32, 2, 1, False),
              ("blk5_tex", 128, 64, 128, 64, 1, 2, True), ("blk4_mesh", 256, 64, 32, 16, 1, 2, True)]
# batch 50 on one GPU, 13 per rank under DDP x4
REC_CASES = [(b, n) for n in (50, 13) for b in REC_BLOCKS]


@pytest.mark.parametrize("blk,N", REC_CASES, ids=[b[0] if n == 50 else f"{b[0]}-N{n}" for b, n in REC_CASES])
def test_reconstruction_block_glue(blk, N):
    """ResBlock.forward_fused's two calls (BatchNorm2d weight / bias shared by the batch, ReLU = slope 0)."""
    name, cin, cout, H, W, up, pad, post = blk
    skip = 'id' if cin == cout else 'sc'
    print(name)
    run_glue(N, [L(cin, H, W, slope=0.0), L(cout, H, W, up, pad, skip, post, slope=0.0)], kind='bn', seed=len(name))


EDGES = {
    "W1_up2": dict(N=4, layers=[L(64, 6, 1, 2, 1, 'id')]),                                 # both pad sides = the one pixel
    "W1_pad2_post": dict(N=3, layers=[L(32, 5, 1, 1, 2, 'sc', True)]),
    "H1": dict(N=8, layers=[L(128, 1, 16, 2, 1, 'sc')]),
    "N1": dict(N=1, layers=[L(64, 12, 10, 2, 1, 'id')]),
    "C4": dict(N=6, layers=[L(4, 16, 8, 2, 1, 'id')]),
    "C1024": dict(N=4, layers=[L(1024, 4, 4, 2, 1, 'id')]),                                # C/4 = 256 = threads per CTA
    "ragged_bwd1_cta": dict(N=32, layers=[L(64, 65, 12, 1, 1, 'sc')]),                     # N*H > 1056, H odd: 2 rows per CTA
    "not_channels_last": dict(N=4, layers=[L(64, 8, 8, 2, 1, 'id')], channels_last=False),
    "near_constant_channel": dict(N=8, layers=[L(16, 8, 8, 2, 1, 'id')], const_channel=True),
    "eval": dict(N=5, layers=[L(64, 8, 6, 2, 1, 'id', True)], training=False),
    "bn_eval": dict(N=5, layers=[L(64, 8, 6, 1, 2, 'sc', True, 0.0)], kind='bn', training=False),
    "bn_near_constant_channel": dict(N=4, layers=[L(32, 6, 5, 2, 1, 'id', False, 0.0)], kind='bn', const_channel=True),
    "bn_eval_without_running_stats": dict(N=6, layers=[L(32, 8, 4, 2, 1, 'id', False, 0.0)], kind='bn', training=False,
                                          bn_kw=dict(track_running_stats=False)),
    "cbn_train_without_running_stats": dict(N=6, layers=[L(32, 8, 4, 2, 1, 'id')], bn_kw=dict(track_running_stats=False)),
    "momentum_none": dict(N=4, layers=[L(16, 4, 4, 1, 1)], bn_kw=dict(momentum=None)),
}


@pytest.mark.parametrize("case", list(EDGES))
def test_glue_edges(case):
    kw = dict(EDGES[case])
    N, layers = kw.pop("N"), kw.pop("layers")
    run_glue(N, layers, seed=7, **kw)


def test_cbn_batch_layers_with_different_widths():
    """Three layers of one CBNBatch with C = 128, 64, 32 (gamma / beta at different column offsets of one GEMM row, one
    gradient sink), chained so that the first layer's backward runs last and closes the sink."""
    run_glue(4, [L(128, 8, 6), L(64, 8, 6), L(32, 8, 6, 2, 1, 'id')], kind='cbn', chain=True, seed=3)


# ---------------------------------------------------------------------------------------------------------------------
# both sources of the statistics
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cin,C,H,W", [(128, 128, 128, 64), (512, 256, 16, 8)])
def test_statistics_from_conv_epilogue_and_from_bn_sums(Cin, C, H, W):
    """cbn_act_pad(sums=) with the sums a conv2d_banked(stats=) epilogue accumulated, and sums=None (b3d_bn_sums), on the
    same conv output: both equal the fp64 glue, and the running buffers follow F.batch_norm."""
    from b3d.bank import WeightBank
    from b3d.conv import conv2d_banked
    from b3d.ew import CBNBatch, cbn_act_pad
    from models.gan import TCConv2d
    torch.manual_seed(C)
    conv = TCConv2d(Cin, C, 3, padding=(1, 0), bias=False).to(DEV)
    Wb = WeightBank({"c": conv}).forward(True)
    x = torch.randn(32, Cin, H, W + 2, device=DEV).contiguous(memory_format=torch.channels_last)
    z = torch.randn(32, EMB, device=DEV)
    cbn_e = make_cbn(C, 11).to(DEV).train()
    cbn_s = copy.deepcopy(cbn_e)
    rm0, rv0 = cbn_e.norm.running_mean.double(), cbn_e.norm.running_var.double()
    with torch.no_grad():
        cb = CBNBatch([cbn_e], z)
        slot = cb.stats_slot(cbn_e)
        y = conv2d_banked(x, Wb["c"], pad_y=1, stats=slot)
        out_e = cbn_act_pad(y, cbn_e, z, up=2, pad=1, cb=cb, sums=slot)
        out_s = cbn_act_pad(y, cbn_s, z, up=2, pad=1)
        ref = {}
        for dt in (torch.float64, torch.float32):
            lin = lambda m: F.linear(z.to(dt), m.weight.to(dt), m.bias.to(dt))
            ref[dt] = ref_glue(y.to(dt), lin(cbn_e.fc_gamma), lin(cbn_e.fc_beta), up=2, pad=1)
    torch.cuda.synchronize()
    o64, o32 = ref[torch.float64][0], ref[torch.float32][0]
    assert_close("out (epilogue sums)", out_e, o64, o32, OUT_CEIL)
    assert_close("out (b3d_bn_sums)", out_s, o64, o32, OUT_CEIL)
    m64, v64 = ref[torch.float64][3], ref[torch.float64][4]
    n = 32 * H * W
    for cbn in (cbn_e, cbn_s):
        rm_ref, rv_ref = 0.9 * rm0 + 0.1 * m64, 0.9 * rv0 + 0.1 * v64 * n / (n - 1)
        assert float((cbn.norm.running_mean.double() - rm_ref).abs().max()) <= 2e-6 * max(1.0, float(rm_ref.abs().max()))
        assert float((cbn.norm.running_var.double() - rv_ref).abs().max()) <= 2e-6 * max(1.0, float(rv_ref.abs().max()))


@pytest.mark.parametrize("N,C,H,W", [(32, 64, 64, 32), (32, 256, 16, 8), (2, 1024, 33, 17)])
@pytest.mark.parametrize("offset,bound", [(16.0, 1e-5), (64.0, 1.5e-4)])
def test_bn_sums_with_large_channel_means(N, C, H, W, offset, bound):
    """Channel means 16x / 64x their standard deviation.  b3d_bn_sums adds fp32 per-thread partials and fp64
    block totals.  On an H100 the largest relative inv_std error over the channels of these shapes is 2.4e-6 at 16x and
    5.7e-5 at 64x (a numpy emulation of the summation order agrees channel by channel in magnitude); the bounds are ~3x
    that.  Adding the block totals in fp32 would miss them by orders of magnitude."""
    from b3d import lib, ptr, stream_ptr
    g = torch.Generator().manual_seed(C + int(offset))
    sd = 0.5 + torch.rand(C, generator=g, dtype=torch.float64)
    y64 = (offset + torch.randn(N, H, W, C, generator=g, dtype=torch.float64)) * sd
    y = y64.float().to(DEV)
    y64 = y.double()
    m_ref, v_ref = y64.mean(dim=(0, 1, 2)), y64.var(dim=(0, 1, 2), unbiased=False)
    inv_ref = (v_ref + EPS).rsqrt()
    sums = torch.empty(2 * C, device=DEV, dtype=torch.float64)
    assert lib.b3d_bn_sums(ptr(y), N * H * W, C, ptr(sums), stream_ptr(y)) == 0
    torch.cuda.synchronize()
    n = N * H * W
    m_s = sums[:C] / n
    inv_s = ((sums[C:] / n - m_s * m_s).clamp(min=0) + EPS).rsqrt()
    rel = float(((inv_s - inv_ref) / inv_ref).abs().max())
    print(f"  b3d_bn_sums offset {offset:g}: rel inv_std error {rel:.2e}")
    assert rel <= bound, f"b3d_bn_sums: relative inv_std error {rel:.2e} > {bound:g}"
    assert float(((m_s - m_ref) / m_ref).abs().max()) <= 1e-6


# ---------------------------------------------------------------------------------------------------------------------
# running buffers across steps
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["bn", "cbn"])
@pytest.mark.parametrize("momentum", [0.1, None], ids=["momentum0.1", "momentumNone"])
def test_running_buffers_follow_batchnorm(kind, momentum):
    """Two training forwards, then eval, against torch's own BatchNorm2d (an fp64 copy of the module): running mean /
    variance and num_batches_tracked after each step, and the eval output from the running statistics.  momentum=None
    is torch's cumulative average (factor 1 / num_batches_tracked)."""
    from b3d.ew import bn_act_pad, cbn_act_pad
    C, N, H, W = 64, 4, 6, 5
    mod = (make_bn(C, 5, momentum=momentum) if kind == 'bn' else make_cbn(C, 5, momentum=momentum)).to(DEV)
    norm = mod if kind == 'bn' else mod.norm
    ref = copy.deepcopy(norm).double()
    g = torch.Generator().manual_seed(9)
    z = torch.randn(N, EMB, generator=g).to(DEV)
    for step, training in enumerate((True, True, False, True)):
        mod.train(training)
        ref.train(training)
        y = (torch.randn(N, C, H, W, generator=g) * (1 + step) + step).to(DEV).contiguous(memory_format=torch.channels_last)
        with torch.no_grad():
            if kind == 'bn':
                out = bn_act_pad(y, mod, up=1, pad=0, slope=0.0)
                want = F.relu(ref(y.double()))
            else:
                out = cbn_act_pad(y, mod, z, up=1, pad=0)
                gam, bet = (F.linear(z.double(), m.weight.double(), m.bias.double())[:, :, None, None]
                            for m in (mod.fc_gamma, mod.fc_beta))
                want = F.leaky_relu(ref(y.double()) * (1 + gam) + bet, 0.2)
        torch.cuda.synchronize()
        err = float((out.double() - want).abs().max())
        assert err <= 2e-6 * float(want.abs().max()), f"step {step}: output differs by {err:.2e}"
        for a, b in ((norm.running_mean, ref.running_mean), (norm.running_var, ref.running_var)):
            e = float((a.double() - b).abs().max())
            assert e <= 2e-6 * max(1.0, float(b.abs().max())), f"step {step}: running buffer differs by {e:.2e}"
        assert int(norm.num_batches_tracked) == int(ref.num_batches_tracked) == (step + 1 if step < 2 else step)


# ---------------------------------------------------------------------------------------------------------------------
# scalar kernels through the C ABI
# ---------------------------------------------------------------------------------------------------------------------
def _f(t):
    return ctypes.c_float(t)


@pytest.mark.parametrize("C", [40, 300])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("momentum", [0.1, -1.0], ids=["momentum0.1", "cumulative"])
def test_cbn_prepare_formulas(C, mode, momentum):
    """b3d_cbn_prepare against the fp64 formulas: mode 0 running statistics, mode 1 F.batch_norm (biased variance + eps,
    clamped at 0), mode 2 the reference's SyncBN (var = (SS - S m) / n, inv_std = clamp(var, eps)^-1/2).  gamma / beta
    live in a wider row (another layer's columns first, gb_pitch > 2C) as in CBNBatch; count = 6 makes the unbiased
    running variance 20 % larger than the biased one; channel 3 is near constant (var ~ eps / 4)."""
    from b3d import lib, ptr, stream_ptr
    N, count, eps, nbt0 = 3, 6.0, EPS, 4
    g = torch.Generator().manual_seed(C + 10 * mode)
    x = torch.randn(int(count), C, generator=g, dtype=torch.float64) * (0.5 + torch.rand(C, generator=g, dtype=torch.float64))
    x = x + torch.randn(C, generator=g, dtype=torch.float64)
    x[:, 3] = 0.3 + (eps / 4) ** 0.5 * torch.randn(int(count), generator=g, dtype=torch.float64)
    sums = torch.cat((x.sum(0), (x * x).sum(0))).to(DEV)
    goff, boff, pitch = 24, 24 + C, 2 * C + 40
    gb = (0.3 * torch.randn(N, pitch, generator=g)).to(DEV)
    rm0 = torch.randn(C, generator=g).to(DEV)
    rv0 = (0.5 + torch.rand(C, generator=g)).to(DEV)
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.full((1,), nbt0, dtype=torch.int64, device=DEV)
    mean, invstd = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    scale, shift, gt = (torch.empty(N, C, device=DEV) for _ in range(3))
    rc = lib.b3d_cbn_prepare(ptr(gb), pitch, goff, boff, ptr(sums), ctypes.c_double(count), _f(eps), _f(momentum), mode,
                             ptr(rm), ptr(rv), ptr(nbt), ptr(mean), ptr(invstd), ptr(scale), ptr(shift), ptr(gt), N, C,
                             stream_ptr(gb))
    assert rc == 0
    torch.cuda.synchronize()
    S, SS = sums[:C], sums[C:]
    if mode == 0:
        m, inv = rm0.double(), (rv0.double() + eps).rsqrt()
    else:
        m = S / count
        var = (SS / count - m * m).clamp(min=0) if mode == 1 else (SS - S * m) / count
        inv = (var + eps).rsqrt() if mode == 1 else var.clamp(min=eps).rsqrt()
    gam, bet = gb[:, goff:goff + C].double(), gb[:, boff:boff + C].double()
    sc = inv[None] * (1 + gam)
    for name, got, want in (("mean", mean, m), ("invstd", invstd, inv), ("scale", scale, sc), ("shift", shift, bet - m[None] * sc),
                            ("gt", gt, 1 + gam)):
        e = float((got.double() - want).abs().max())
        assert e <= 1e-6 * max(1.0, float(want.abs().max())), f"{name} differs by {e:.2e}"
    if mode == 0:                                              # eval: buffers read, never written
        assert torch.equal(rm, rm0) and torch.equal(rv, rv0) and int(nbt) == nbt0
        return
    f = momentum if momentum >= 0 else 1.0 / (nbt0 + 1)
    rm_ref = (1 - f) * rm0.double() + f * m
    rv_ref = (1 - f) * rv0.double() + f * var * count / (count - 1)
    assert float((rm.double() - rm_ref).abs().max()) <= 1e-6 * max(1.0, float(rm_ref.abs().max()))
    assert float((rv.double() - rv_ref).abs().max()) <= 1e-6 * max(1.0, float(rv_ref.abs().max()))
    assert int(nbt) == nbt0 + 1


def test_cbn_bwd_reduce_uses_per_sample_gamma():
    """b3d_cbn_bwd_reduce: red[0] = sum_n (1 + gamma[n]) S1[n], red[1] = sum_n (1 + gamma[n]) S2[n] with the per-sample
    sums in rows of pitch s_pitch > C (the slices of the d(gamma, beta) sink); the columns beyond C are never read."""
    from b3d import lib, ptr, stream_ptr
    N, C, pitch = 7, 44, 72
    g = torch.Generator().manual_seed(2)
    S1, S2 = (torch.randn(N, pitch, generator=g).to(DEV) for _ in range(2))
    S1[:, C:] = float("nan")
    S2[:, C:] = float("nan")
    gt = (1 + 0.4 * torch.randn(N, C, generator=g)).to(DEV)
    red = torch.empty(2 * C, device=DEV)
    assert lib.b3d_cbn_bwd_reduce(ptr(S1), ptr(S2), pitch, ptr(gt), ptr(red), N, C, stream_ptr(gt)) == 0
    torch.cuda.synchronize()
    want = torch.cat(((gt.double() * S1[:, :C].double()).sum(0), (gt.double() * S2[:, :C].double()).sum(0)))
    e = float((red.double() - want).abs().max())
    assert e <= 1e-6 * float(want.abs().max()), f"red differs by {e:.2e}"


@pytest.mark.parametrize("C", [12, 1040])
@pytest.mark.parametrize("up,pad,post", [(2, 1, False), (1, 2, True)])
@pytest.mark.parametrize("pad_mode", [0, 1])
def test_cbn_act_fwd_generic_kernel_pad_modes(pad_mode, C, up, pad, post):
    """b3d_cbn_act_fwd where C/4 does not divide 256 (the generic grid-stride kernel, include/b3d.h allows any C % 4 == 0):
    out = post(leaky(y * scale + shift) + skip[x + skip_off]) upsampled and x-padded (pad_mode 0 replicate, 1 circular in
    upsampled columns), skip with a row pitch W + 3."""
    from b3d import lib, ptr, stream_ptr
    N, H, W, off, slope = 3, 5, 7, 2, 0.2
    g = torch.Generator().manual_seed(C + up)
    y = torch.randn(N, H, W, C, generator=g).to(DEV)
    scale = (1 + 0.3 * torch.randn(N, C, generator=g)).to(DEV)
    shift = (0.3 * torch.randn(N, C, generator=g)).to(DEV)
    skip = torch.randn(N, H, W + 3, C, generator=g).to(DEV)
    out = torch.empty(N, up * H, up * W + 2 * pad, C, device=DEV)
    assert lib.b3d_cbn_act_fwd(ptr(y), ptr(scale), ptr(shift), ptr(skip), W + 3, off, ptr(out), N, H, W, C, up, pad, pad_mode,
                               _f(slope), int(post), stream_ptr(y)) == 0
    torch.cuda.synchronize()
    h = F.leaky_relu(y.double() * scale.double()[:, None, None] + shift.double()[:, None, None], slope) \
        + skip.double()[:, :, off:off + W]
    if post:
        h = F.leaky_relu(h, slope)
    h = h.permute(0, 3, 1, 2)
    if up == 2:
        h = F.interpolate(h, scale_factor=2, mode='nearest')
    want = (F.pad(h, (pad, pad, 0, 0), mode='replicate') if pad_mode == 0 else
            torch.cat((h[..., -pad:], h, h[..., :pad]), dim=3)).permute(0, 2, 3, 1)
    e = float((out.double() - want).abs().max())
    assert e <= 1e-6 * float(want.abs().max()), f"generic cbn_act_fwd differs by {e:.2e}"


# ---------------------------------------------------------------------------------------------------------------------
# block wiring: forward_fused == forward + upsample + pad on the same convolutions
# ---------------------------------------------------------------------------------------------------------------------
WIRING_TOL = 1e-3


def _wiring_compare(fused, plain, leaves_f, leaves_p, params_f, params_p, norms_f, norms_p):
    for name, a, b in [("out", fused, plain)] + [(f"d leaf{i}", x.grad, y.grad) for i, (x, y) in enumerate(zip(leaves_f, leaves_p))] \
            + [(n, p.grad, q.grad) for (n, p), q in zip(params_f, params_p)]:
        e = float((a.double() - b.double()).abs().max()) / float(b.double().abs().max())
        print(f"  {name:24s} rel {e:.2e}")
        assert e <= WIRING_TOL, f"{name}: fused and unfused blocks differ by {e:.2e} of the largest magnitude"
    for nf, np_ in zip(norms_f, norms_p):
        assert torch.allclose(nf.running_mean, np_.running_mean, rtol=1e-4, atol=1e-5)
        assert torch.allclose(nf.running_var, np_.running_var, rtol=1e-4, atol=1e-5)
        assert int(nf.num_batches_tracked) == int(np_.num_batches_tracked) == 1


@pytest.mark.parametrize("cin,cout,up,pad,post", [(128, 64, 1, 2, True), (128, 128, 2, 1, False)])
def test_generator_block_wiring(cin, cout, up, pad, post):
    """ResBlockUp.forward_fused(W=None) against forward + LeakyReLU + upsample + pad on the same modules (spectral norm
    removed so that both paths see identical weights).  Both use the same tf32 convolutions; the fused path feeds conv2 the
    kernel's output instead of torch's, and tf32 rounding of those slightly different inputs is what remains (at most
    1.5e-4 of the largest magnitude measured on an H100, in a weight gradient): the bound is 1e-3."""
    from b3d.ew import CBNBatch, REPLICATE, pad_x
    from models.gan import ResBlockUp
    torch.manual_seed(cin + cout)
    args = types.SimpleNamespace(norm_g='batch')
    padf = lambda t, a: pad_x(t, a, REPLICATE)
    blk = ResBlockUp(args, cin, cout, EMB, padf)
    for m in (blk.conv1, blk.conv2, blk.shortcut):
        if isinstance(m, torch.nn.Module):
            torch.nn.utils.remove_spectral_norm(m)
    for cbn in (blk.norm1, blk.norm2):
        with torch.no_grad():
            cbn.fc_gamma.weight.normal_(0, 0.3 / EMB ** 0.5)
            cbn.fc_beta.weight.normal_(0, 0.3 / EMB ** 0.5)
    blk = blk.to(DEV).train()
    blk_p = copy.deepcopy(blk)
    x = torch.randn(8, cin, 16, 8, device=DEV).contiguous(memory_format=torch.channels_last)
    z = torch.randn(8, EMB, device=DEV)
    xf, zf, xp_, zp = (t.clone().requires_grad_(True) for t in (x, z, x, z))
    cb = CBNBatch([blk.norm1, blk.norm2], zf)
    fused = blk.forward_fused(padf(xf, 1), zf, up, pad, post_leaky=post, cb=cb)
    h = blk_p(xp_, zp)
    if post:
        h = F.leaky_relu(h, 0.2)
    if up == 2:
        h = F.interpolate(h, scale_factor=2, mode='nearest')
    plain = F.pad(h, (pad, pad, 0, 0), mode='replicate')
    w = torch.randn(plain.shape, device=DEV)
    (fused * w).sum().backward()
    (plain * w).sum().backward()
    torch.cuda.synchronize()
    _wiring_compare(fused.detach(), plain.detach(), [xf, zf], [xp_, zp], list(blk.named_parameters()),
                    [p for _, p in blk_p.named_parameters()], [blk.norm1.norm, blk.norm2.norm], [blk_p.norm1.norm, blk_p.norm2.norm])


@pytest.mark.parametrize("cin,cout,up,pad,post", [(128, 64, 1, 2, True), (256, 256, 2, 1, False)])
def test_reconstruction_block_wiring(cin, cout, up, pad, post):
    """ResBlock.forward_fused against forward + ReLU + upsample + pad on the same modules (bound as above)."""
    from b3d.ew import REPLICATE, pad_x
    from models.reconstruction import ResBlock
    torch.manual_seed(cin + cout)
    padf = lambda t, a: pad_x(t, a, REPLICATE)
    blk = ResBlock(cin, cout, padf)
    with torch.no_grad():
        for bn in (blk.bn1, blk.bn2):
            bn.weight.uniform_(0.6, 1.4)
            bn.bias.normal_(0, 0.2)
    blk = blk.to(DEV).train()
    blk_p = copy.deepcopy(blk)
    x = torch.randn(6, cin, 16, 8, device=DEV).contiguous(memory_format=torch.channels_last)
    xf, xp_ = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    fused = blk.forward_fused(padf(xf, 1), up, pad, post_relu=post)
    h = blk_p(xp_)
    if post:
        h = F.relu(h)
    if up == 2:
        h = F.interpolate(h, scale_factor=2, mode='nearest')
    plain = F.pad(h, (pad, pad, 0, 0), mode='replicate')
    w = torch.randn(plain.shape, device=DEV)
    (fused * w).sum().backward()
    (plain * w).sum().backward()
    torch.cuda.synchronize()
    _wiring_compare(fused.detach(), plain.detach(), [xf], [xp_], list(blk.named_parameters()),
                    [p for _, p in blk_p.named_parameters()], [blk.bn1, blk.bn2], [blk_p.bn1, blk_p.bn2])
